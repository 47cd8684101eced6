"""The fused allreduce+SGD and allreduce+LARS steps held bit for bit to the exact oracle of tests/optimizer_oracle.py.

The kernels run on a world-1 real communicator and on emulated communicators of 1-8 virtual ranks (one launch, gridDim.y ==
world). Every case runs three steps, each checked against the oracle applied to the kernel's own previous parameters and
momentum, so an error cannot hide behind an earlier one; step 0 is a first step over a NaN-filled momentum, which must not
be read. Parameters, momentum, the bf16 shadow and LARS's trust ratios are compared bitwise on every rank (a NaN matches any
NaN); the bytes around the region in the parameter, shadow and gradient windows and past every momentum shard must not
change. LARS trust ratios are exact where the norm sums are exact in any order (the exact-norm family) and otherwise
bounded (the random family); the update is exact given the kernel's own trust ratios."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from collective_oracle import assert_bits
from ema_oracle import ema_step
from optimizer_oracle import (F32, expand_groups, lars_norm_interval, lars_step, owner_sum, sgd_step, vec_elems)

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD_VECS = 16                  # vectors after the region in every window, and floats after every momentum shard
OFF_VECS = 24                    # the region starts this many vectors into its windows
SENT = -7.25
STEPS = [(0.1, 0.9, 1e-4), (0.05, 0.5, 1e-2), (0.2, 0.0, 0.0)]
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def _real_comm(tag):
    from mpi_operator_b200.runtime.comm import Communicator
    return Communicator.create(0, 1, 0, f"t-optx-{tag}-{os.getpid()}")


@pytest.fixture(scope="module", params=["real1", 1, 2, 3, 4, 5, 6, 7, 8])
def comm(request):
    from mpi_operator_b200.runtime.comm import Communicator
    c = _real_comm("k") if request.param == "real1" else Communicator.local(request.param, device=0)
    c.set_tuning(timeout_ms=5000)
    yield c
    c.set_hyper(None)
    c.destroy()


def _one(comm, xs):
    return xs if comm.is_local else xs[0]


def _np(t):
    return t.detach().float().cpu().numpy()


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


class Bucket:
    """One region of ``n`` gradient elements of ``gdtype`` (and ``n`` fp32 parameters, ``n`` bf16 shadows), OFF_VECS vectors
    into windows that end GUARD_VECS vectors after it; momentum (and EMA) shards are views into buffers with a tail. The
    optional LARS layout is a list of (elements, group, lars) parameters; vectors after them carry the tail key P."""

    def __init__(self, comm, n, gdtype=torch.float32, layout=None, table=None):
        self.comm, self.W, self.n, self.gdtype = comm, comm.world, n, gdtype
        N = vec_elems(gdtype)
        self.N, self.esz = N, torch.empty((), dtype=gdtype).element_size()
        self.lo, tot = OFF_VECS * N, (OFF_VECS + GUARD_VECS) * N + n
        self.gwin = comm.alloc_window(tot * self.esz)
        self.pwin, self.lwin = comm.alloc_window(tot * 4), comm.alloc_window(tot * 2)
        self.gfull = self._per_rank(self.gwin, gdtype, tot)
        self.pfull = self._per_rank(self.pwin, torch.float32, tot)
        self.lfull = self._per_rank(self.lwin, torch.bfloat16, tot)
        sl = slice(self.lo, self.lo + n)
        self.gv, self.pv, self.lv = [g[sl] for g in self.gfull], [p[sl] for p in self.pfull], [x[sl] for x in self.lfull]
        self.per = comm.slice_elems(n, gdtype)
        self.mbuf = [torch.full((self.per + GUARD_VECS,), SENT, device="cuda") for _ in range(self.W)]
        self.moms = [b[:self.per] for b in self.mbuf]
        self.ebuf = [torch.full((self.per + GUARD_VECS,), SENT, device="cuda") for _ in range(self.W)]
        self.emas = [b[:self.per] for b in self.ebuf]
        self.sched = torch.tensor([float(np.float32(0.99)), 0.0], dtype=torch.float64, device="cuda")
        for w in (self.gfull, self.pfull, self.lfull):         # random bytes everywhere: guards, and the region until set
            for t in w:
                t.view(torch.uint8).copy_(torch.randint(0, 256, (t.numel() * t.element_size(),), dtype=torch.uint8))
        self.layout, self.table = layout, table
        if layout is not None:
            P = len(layout)
            pmap = np.full(n // 4, P, dtype=np.int32)
            self.slots, s = [], 0
            for k, (ne, _, _) in enumerate(layout):
                nv = -(-ne // 4)
                pmap[s:s + nv] = k
                self.slots.append((4 * s, 4 * (s + nv)))
                s += nv
            assert s <= n // 4
            self.pmap_np = pmap
            self.pmap = torch.from_numpy(pmap).to(torch.uint16).cuda()
            self.ptab = torch.tensor([[g, l] for _, g, l in layout], dtype=torch.uint8, device="cuda")
            self.board = comm.alloc_window(P * self.W * 8 + 16)
            nb = comm.lars_scratch_bytes(n, P)
            self.scratch = [torch.zeros(nb, dtype=torch.uint8, device="cuda") for _ in range(self.W)]
            self.trust = [torch.full((P,), NAN, device="cuda") for _ in range(self.W)]

    def _per_rank(self, win, dtype, numel):
        if self.comm.is_local:
            return [win.tensor(dtype, rank=r, numel=numel) for r in range(self.W)]
        return [win.tensor(dtype, numel=numel)]

    def live(self, r):
        return max(0, min(self.per, self.n - r * self.per))

    # ---------------------------------------------------------------------------------------------- state --
    def set_params(self, p):
        for v in self.pv:
            v.copy_(_t(p))

    def set_grads(self, gs):
        """gs: one fp32 numpy array per rank, already representable in gdtype."""
        for v, g in zip(self.gv, gs):
            v.copy_(_t(g).to(self.gdtype))

    def momentum(self):
        return np.concatenate([_np(self.moms[r][:self.live(r)]) for r in range(self.W)])

    def ema(self):
        return np.concatenate([_np(self.emas[r][:self.live(r)]) for r in range(self.W)])

    def seal(self):
        """Record every byte the step may not write: the windows outside the region, all gradients, the shard tails."""
        self.snap = [t.clone() for t in self.gfull] + [torch.cat([t[:self.lo], t[self.lo + self.n:]]).clone()
                                                       for t in self.pfull + self.lfull]
        self.snap_m = [b[self.live(r):].clone() for r, b in enumerate(self.mbuf)]
        self.snap_e = [b[self.live(r):].clone() for r, b in enumerate(self.ebuf)]

    def check_bounds(self, what):
        now = [t for t in self.gfull] + [torch.cat([t[:self.lo], t[self.lo + self.n:]]) for t in self.pfull + self.lfull]
        for a, b in zip(now, self.snap):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{what}: a write outside the region"
        for r in range(self.W):
            for buf, snap in ((self.mbuf, self.snap_m), (self.ebuf, self.snap_e)):
                assert torch.equal(buf[r][self.live(r):].view(torch.int32), snap[r].view(torch.int32)), \
                    f"{what}: rank {r} wrote past its live shard"

    # --------------------------------------------------------------------------------------------- launch --
    def sgd(self, lr, mu, wd, nesterov, first, scale=None, groups=None, ema=False):
        c = self.comm
        kw = dict(ema=_one(c, self.emas), ema_sched=self.sched) if ema else {}
        if groups is not None:
            kw.update(group_map=groups[0], group_hyper=groups[1])
        c.allreduce_sgd_window(self.gwin, self.lo * self.esz, self.pwin, self.lo * 4, _one(c, self.moms), self.n,
                               self.gdtype, lr=lr, momentum_coef=mu, weight_decay=wd, nesterov=nesterov, first_step=first,
                               scale=scale, lowp_win=self.lwin, lowp_off=self.lo * 2, algo="twoshot", **kw)

    def lars(self, eta, nesterov, first, scale=None, ema=False):
        c = self.comm
        kw = dict(ema=_one(c, self.emas), ema_sched=self.sched) if ema else {}
        c.allreduce_lars_window(self.gwin, self.lo * 4, self.pwin, self.lo * 4, _one(c, self.moms), self.n, torch.float32,
                                group_hyper=self.table, param_map=self.pmap, param_table=self.ptab, board_win=self.board,
                                board_off=0, scratch=_one(c, self.scratch), trust_coefficient=eta, nesterov=nesterov,
                                first_step=first, scale=scale, lowp_win=self.lwin, lowp_off=self.lo * 2, algo="twoshot",
                                trust_out=_one(c, self.trust), **kw)

    # ---------------------------------------------------------------------------------------------- check --
    def check(self, want_p, want_m, want_sh, what):
        torch.cuda.synchronize()
        self.comm.check_error()
        wp = _t(want_p)
        wsh = _t(want_sh.view(np.int16)).view(torch.bfloat16)
        for r in range(self.W):
            assert_bits(self.pv[r].cpu(), wp, f"{what}: parameters rank {r}")
            assert_bits(self.lv[r].cpu(), wsh, f"{what}: bf16 shadow rank {r}")
        assert_bits(_t(self.momentum()), _t(want_m), f"{what}: momentum")
        self.check_bounds(what)

    def free(self):
        for w in (self.gwin, self.pwin, self.lwin):
            w.free()
        if self.layout is not None:
            self.board.free()


def _params(rng, n):
    """Parameters over 2^+-8 with zeros, subnormals and bf16 rounding ties mixed in."""
    p = (rng.standard_normal(n) * 2.0 ** rng.integers(-8, 9, n)).astype(F32)
    k = np.arange(n)
    p[k % 13 == 1] = (1 + 2.0 ** -8) * 2.0 ** rng.integers(-4, 4, int((k % 13 == 1).sum()))     # ties: stay at even
    p[k % 13 == 2] = -(1 + 3 * 2.0 ** -8)                                                        # ties: round up
    p[k % 13 == 3] = (rng.integers(1, 1 << 20, int((k % 13 == 3).sum())) * 2.0 ** -149).astype(F32)   # subnormal
    p[k % 13 == 4] = 0.0
    return p


def _grads(rng, W, n, dtype, scale=2.0 ** -4):
    """Per-rank gradients representable in ``dtype`` (fp32 arrays), with subnormals (fp32 and bf16 range) mixed in."""
    out = []
    for _ in range(W):
        g = (rng.standard_normal(n) * scale * 2.0 ** rng.integers(-6, 4, n)).astype(F32)
        k = np.arange(n)
        g[k % 13 == 3] = (rng.integers(-(1 << 12), 1 << 12, int((k % 13 == 3).sum())) * 2.0 ** -140).astype(F32)
        out.append(_np(_t(g).to(dtype)))
    return out


def _scale(comm, scale):
    return F32(1.0 / comm.world) if scale is None else F32(scale)


# ------------------------------------------------------------------------------------------------- SGD, ungrouped --
@pytest.mark.parametrize("hyper, scale", [("value", None), ("device", None), ("value", 0.37)],
                         ids=["value-avg", "device-avg", "value-scale"])
@pytest.mark.parametrize("nesterov", [False, True], ids=["plain", "nesterov"])
@pytest.mark.parametrize("gdtype", DTYPES, ids=lambda d: str(d)[6:])
def test_sgd_exact(comm, gdtype, nesterov, hyper, scale):
    """k_allreduce_sgd<T, P2P>: 1013 vectors (ragged slices at every world). With hyper="device" the kernel reads
    {lr, mu, wd} from the set_hyper table, which changes between steps, and the by-value arguments are wrong."""
    W, N = comm.world, vec_elems(gdtype)
    n = 1013 * N
    rng = np.random.default_rng(W * 1000 + DTYPES.index(gdtype) * 100 + nesterov * 10 + (hyper == "device") * 2 + (scale is None))
    B = Bucket(comm, n, gdtype)
    table = torch.zeros(3, device="cuda")
    try:
        B.set_params(_params(rng, n))
        for r in range(W):
            B.moms[r].fill_(NAN)
        if hyper == "device":
            comm.set_hyper(table)
        for step, (lr, mu, wd) in enumerate(STEPS):
            gs = _grads(rng, W, n, gdtype)
            B.set_grads(gs)
            p, m = _np(B.pv[0]), B.momentum()
            B.seal()
            if hyper == "device":
                table.copy_(torch.tensor([lr, mu, wd]))
                B.sgd(7.0, 0.25, 0.5, nesterov, step == 0, scale)
            else:
                B.sgd(lr, mu, wd, nesterov, step == 0, scale)
            S = owner_sum(gs, W, gdtype)
            want = sgd_step(p, m, S, _scale(comm, scale), F32(lr), F32(mu), F32(wd), nesterov, step == 0)
            B.check(*want, f"step {step}")
    finally:
        comm.set_hyper(None)
        B.free()


# --------------------------------------------------------------------------------------------------- SGD, grouped --
def _group_table(rng):
    """256 rows of {lr, mu, wd}; lr = 0 (frozen), mu = 0 and wd = 0 on rows of their own."""
    t = np.stack([rng.uniform(0, 0.5, 256), rng.uniform(0, 0.99, 256), rng.uniform(0, 1e-2, 256)], 1).astype(F32)
    k = np.arange(256)
    t[k % 7 == 0, 0] = 0
    t[k % 5 == 0, 1] = 0
    t[k % 3 == 0, 2] = 0
    return t


@pytest.mark.parametrize("nesterov", [False, True], ids=["plain", "nesterov"])
def test_grouped_sgd_exact(comm, nesterov):
    """k_allreduce_sgd<float, P2P, true>: a 256-row table that changes every step, the map cycling through every row; a
    set_hyper table and the by-value arguments are present and must be ignored."""
    W, n = comm.world, 4 * 1013
    rng = np.random.default_rng(W * 7 + nesterov)
    B = Bucket(comm, n)
    gmap_np = (np.arange(n // 4) % 256).astype(np.uint8)
    gmap, ghyper = torch.from_numpy(gmap_np).cuda(), torch.zeros(256, 3, device="cuda")
    wrong = torch.tensor([3.0, 0.5, 0.25], device="cuda")
    try:
        comm.set_hyper(wrong)
        B.set_params(_params(rng, n))
        for r in range(W):
            B.moms[r].fill_(NAN)
        for step in range(3):
            tab = _group_table(rng)
            ghyper.copy_(_t(tab))
            gs = _grads(rng, W, n, torch.float32)
            B.set_grads(gs)
            p, m = _np(B.pv[0]), B.momentum()
            B.seal()
            B.sgd(9.0, 9.0, 9.0, nesterov, step == 0, groups=(gmap, ghyper))
            lr, mu, wd = expand_groups(tab, gmap_np, n)
            want = sgd_step(p, m, owner_sum(gs, W, torch.float32), _scale(comm, None), lr, mu, wd, nesterov, step == 0)
            B.check(*want, f"step {step}")
            frozen = lr == 0
            assert np.array_equal(_np(B.pv[0])[frozen], p[frozen])        # lr = 0: the parameters keep their values
    finally:
        comm.set_hyper(None)
        B.free()


# ---------------------------------------------------------------------------------------------------------- LARS --
# (elements, group, lars, kind); kind: the gradients and weights the parameter gets
LARS_LAYOUT = [(4, 0, 1, "rand"), (4 * 3001, 0, 1, "rand"), (4 * 37, 1, 0, "rand"), (4 * 64, 0, 1, "zero_w"),
               (4 * 64, 1, 1, "zero_g"), (4 * 50, 0, 1, "tiny"), (4 * 50, 1, 1, "huge"), (4 * 129, 1, 1, "rand")]
LARS_TAIL = 4 * 5
ETA = 0.02


def _lars_tab(rng):
    """Weight decays large enough that wd * |w| is of the order of |g|: its rounding then shows in the trust ratio."""
    return np.array([[0.5, 0.9, 0.5], [rng.uniform(0.01, 0.5), rng.uniform(0, 0.99), rng.uniform(0.1, 1)]], dtype=F32)


def _lars_inputs(rng, B, layout, exact):
    """Weights and per-rank gradients of every parameter. The exact family puts both on small grids, so every order of the
    norm sums is exact (with scale = 1/world a power of two)."""
    W, n = B.W, B.n
    p = _params(rng, n) if not exact else (rng.integers(-31, 32, n) * 2.0 ** -8).astype(F32)
    gs = [(rng.standard_normal(n) * 2.0 ** rng.integers(-8, 0, n)).astype(F32) for _ in range(W)] if not exact else \
        [(rng.integers(-3, 4, n) * 2.0 ** -6).astype(F32) for _ in range(W)]
    for (s, e), (_, _, _, kind) in zip(B.slots, layout):
        if kind == "zero_w":
            p[s:e] = 0
        for g in gs:
            if kind == "zero_g":
                g[s:e] = 0
            elif kind == "tiny":
                g[s:e] = (rng.uniform(0.5, 1, e - s) * 1e-24).astype(F32)     # (gs)^2 < 2^-150: sg rounds to 0
            elif kind == "huge":
                g[s:e] = (rng.uniform(0.5, 1, e - s) * 1e20).astype(F32)      # (gs)^2 > fp32 max: sg = inf
    return p, gs


def _check_trust(B, layout, S, scale, p, tab, exact, what):
    """Every rank's trust ratios are the same bits; each lies in the oracle's interval (one value when exact)."""
    trust = [_np(t) for t in B.trust]
    for r in range(1, B.W):
        assert np.array_equal(trust[r].view(np.int32), trust[0].view(np.int32)), f"{what}: rank {r} trust differs"
    gsc = (S * scale).astype(F32)
    for k, ((s, e), (_, grp, lars, kind)) in enumerate(zip(B.slots, layout)):
        t = float(trust[0][k])
        if not lars or kind in ("zero_w", "zero_g", "tiny"):
            lo = hi = 1.0
        elif kind == "huge":
            lo = hi = 0.0
        else:
            lo, hi = lars_norm_interval(gsc[s:e], p[s:e], B.W, F32(ETA), tab[grp, 2], exact=exact)
        assert lo <= t <= hi, f"{what}: parameter {k} ({kind}) trust {t!r} not in [{lo!r}, {hi!r}]"
    return trust[0]


def _lars_want(B, layout, trust, p, m, S, scale, tab, nesterov, first):
    """The update given the kernel's trust ratios, expanded to elements (tail vectors: trust 1, group 0)."""
    key = np.repeat(B.pmap_np, 4)[:B.n]
    grp = np.array([g for _, g, _, _ in layout] + [0])[key]
    t = np.append(trust, F32(1.0))[key].astype(F32)
    return lars_step(p, m, S, scale, t, tab[grp, 0], tab[grp, 1], tab[grp, 2], nesterov, first)


def _run_lars(comm, layout, tail, exact, nesterov, seed, ema=False, steps=3):
    W = comm.world
    n = sum(-(-e // 4) * 4 for e, *_ in layout) + tail
    rng = np.random.default_rng(seed)
    table = torch.zeros(2, 3, device="cuda")
    B = Bucket(comm, n, layout=[(e, g, lr) for e, g, lr, _ in layout], table=table)
    scale = _scale(comm, None)
    try:
        p, _ = _lars_inputs(rng, B, layout, exact)
        B.set_params(p)
        for r in range(W):
            B.moms[r].fill_(NAN)
        e_old = None
        for step in range(steps):
            tab = _lars_tab(rng)
            table.copy_(_t(tab))
            p_new, gs = _lars_inputs(rng, B, layout, exact)
            if not exact:                              # the kernel's own parameters, zero-weight tensors kept at zero
                p_new = _np(B.pv[0])
                for (s, e), (_, _, _, kind) in zip(B.slots, layout):
                    if kind == "zero_w":
                        p_new[s:e] = 0
            B.set_params(p_new)                        # exact family: back on the grid, so the norm sums stay exact
            B.set_grads(gs)
            p, m = _np(B.pv[0]), B.momentum()
            if ema:
                e_old = B.ema()
                B.sched[1:].add_(1)
            B.seal()
            B.lars(ETA, nesterov, step == 0, ema=ema)
            torch.cuda.synchronize()
            comm.check_error()
            S = owner_sum(gs, W, torch.float32)
            trust = _check_trust(B, layout, S, scale, p, tab, exact, f"step {step}")
            want = _lars_want(B, layout, trust, p, m, S, scale, tab, nesterov, step == 0)
            B.check(*want, f"step {step}")
            if ema:
                assert_bits(_t(B.ema()), _t(ema_step(e_old, want[0], 0.99, step + 1)), f"step {step}: average")
    finally:
        B.free()


@pytest.mark.parametrize("nesterov", [False, True], ids=["plain", "nesterov"])
def test_lars_exact_norms(comm, nesterov):
    """Norm sums exact in any order (worlds 1, 2, 4, 8: scale = 1/world is a power of two): trust and update bit for bit."""
    if comm.world not in (1, 2, 4, 8):
        pytest.skip("the exact-norm family needs a power-of-two world")
    _run_lars(comm, LARS_LAYOUT, LARS_TAIL, True, nesterov, seed=comm.world)


@pytest.mark.parametrize("nesterov", [False, True], ids=["plain", "nesterov"])
def test_lars_random(comm, nesterov):
    """Random gradients and weights: trust inside the oracle's interval and the same on every rank; the update exact given
    that trust; non-LARS, zero-weight, zero-gradient and underflowing parameters exactly 1, overflowing ones exactly 0."""
    _run_lars(comm, LARS_LAYOUT, LARS_TAIL, False, nesterov, seed=100 + comm.world)


def test_lars_one_vector_parameters(comm):
    """1024 one-vector parameters: the segmented warp scan changes key on every lane. Exact-norm family at worlds 1, 2, 4
    and 8 (683 trust ratios checked bit for bit per step), random family at the others."""
    layout = [(4, k % 2, int(k % 3 != 0), "rand") for k in range(1024)]
    _run_lars(comm, layout, 4 * 3, comm.world in (1, 2, 4, 8), False, seed=200 + comm.world)


# ----------------------------------------------------------------------------------------------------------- EMA --
@pytest.mark.parametrize("kind", ["sgd", "grouped", "lars"])
def test_ema_instantiations_update_exact(comm, kind):
    """The EMA instantiations (fp32 SGD, grouped SGD, LARS): p' and m' bit for bit, and the average from them."""
    if kind == "lars":
        _run_lars(comm, LARS_LAYOUT[:3] + LARS_LAYOUT[5:], LARS_TAIL, False, True, seed=300 + comm.world, ema=True)
        return
    W, n = comm.world, 4 * 1013
    rng = np.random.default_rng(400 + W)
    B = Bucket(comm, n)
    gmap_np = (np.arange(n // 4) % 256).astype(np.uint8)
    gmap, ghyper = torch.from_numpy(gmap_np).cuda(), torch.zeros(256, 3, device="cuda")
    try:
        p0 = _params(rng, n)
        B.set_params(p0)
        for r in range(W):
            B.moms[r].fill_(NAN)
            B.emas[r][:B.live(r)].copy_(_t(p0[r * B.per:r * B.per + B.live(r)]))
        for step, (lr, mu, wd) in enumerate(STEPS):
            gs = _grads(rng, W, n, torch.float32)
            B.set_grads(gs)
            p, m, e = _np(B.pv[0]), B.momentum(), B.ema()
            B.sched[1:].add_(1)
            B.seal()
            S = owner_sum(gs, W, torch.float32)
            if kind == "grouped":
                tab = _group_table(rng)
                ghyper.copy_(_t(tab))
                B.sgd(9.0, 9.0, 9.0, True, step == 0, groups=(gmap, ghyper), ema=True)
                want = sgd_step(p, m, S, _scale(comm, None), *expand_groups(tab, gmap_np, n), True, step == 0)
            else:
                B.sgd(lr, mu, wd, True, step == 0, ema=True)
                want = sgd_step(p, m, S, _scale(comm, None), F32(lr), F32(mu), F32(wd), True, step == 0)
            B.check(*want, f"step {step}")
            assert_bits(_t(B.ema()), _t(ema_step(e, want[0], 0.99, step + 1)), f"step {step}: average")
    finally:
        B.free()


# ------------------------------------------------------------------------------------------------------ geometry --
@pytest.mark.parametrize("blocks", [1, 3, 0], ids=["1cta", "3cta", "default"])
@pytest.mark.parametrize("nvec", [1, 3, 1013, 2359296 // 4], ids=["1vec", "3vec", "1013vec", "resnet"])
@pytest.mark.parametrize("kind", ["sgd", "lars"])
def test_geometry(comm, kind, nvec, blocks):
    """One vector, fewer vectors than ranks (empty slices), ragged slices and a ResNet-size tensor (2,359,296 elements,
    default grid, the real communicator and 8 virtual ranks), on grids forced to 1 and 3 CTAs and the default."""
    if nvec > 1013 and (blocks or comm.world not in (1, 8)):
        pytest.skip("the ResNet-size tensor runs on the default grid at worlds 1 and 8")
    old = comm.get_tuning()["max_blocks"]
    try:
        if blocks:
            comm.set_tuning(max_blocks=blocks)
        if kind == "lars":
            layout = [(4 * max(1, nvec - 2), 0, 1, "rand")] + ([(4, 1, 1, "rand")] if nvec >= 3 else [])
            tail = 4 * (nvec - sum(-(-e // 4) for e, *_ in layout))
            _run_lars(comm, layout, tail, False, True, seed=nvec + blocks, steps=2 if nvec > 1013 else 3)
            return
        W, n = comm.world, 4 * nvec
        rng = np.random.default_rng(nvec * 3 + blocks)
        B = Bucket(comm, n)
        try:
            B.set_params(_params(rng, n))
            for r in range(W):
                B.moms[r].fill_(NAN)
            for step, (lr, mu, wd) in enumerate(STEPS):
                gs = _grads(rng, W, n, torch.float32)
                B.set_grads(gs)
                p, m = _np(B.pv[0]), B.momentum()
                B.seal()
                B.sgd(lr, mu, wd, False, step == 0)
                want = sgd_step(p, m, owner_sum(gs, W, torch.float32), _scale(comm, None), F32(lr), F32(mu), F32(wd),
                                False, step == 0)
                B.check(*want, f"step {step}")
        finally:
            B.free()
    finally:
        comm.set_tuning(max_blocks=old)


# ---------------------------------------------------------------------------------------------------- non-finite --
@pytest.mark.parametrize("kind", ["sgd", "lars"])
def test_nan_and_inf_gradient_on_one_rank(comm, kind):
    """A NaN gradient on the last rank and an Inf on rank 0: NaN / Inf only in those elements' parameters and momentum;
    in LARS the NaN tensor's trust is 1 (NaN norm) and the Inf tensor's 0 (infinite norm); everything else exact."""
    W = comm.world
    layout = [(4 * 40, 0, 1), (4 * 40, 1, 1), (4 * 40, 0, 0)]
    n = 4 * 120
    rng = np.random.default_rng(500 + W)
    tab = np.array([[0.5, 0.9, 1e-3], [0.1, 0.5, 1e-2]], dtype=F32)
    table = torch.from_numpy(tab).cuda()
    B = Bucket(comm, n, layout=layout if kind == "lars" else None, table=table)
    ia, ib = 4 * 5 + 1, 4 * 40 + 4 * 7 + 2              # one element in each of the first two parameters
    try:
        B.set_params(_params(rng, n))
        for r in range(W):
            B.moms[r].fill_(NAN)
        for step in range(3):
            gs = _grads(rng, W, n, torch.float32)
            gs[W - 1][ia], gs[0][ib] = NAN, np.inf
            B.set_grads(gs)
            p, m = _np(B.pv[0]), B.momentum()
            B.seal()
            S = owner_sum(gs, W, torch.float32)
            if kind == "lars":
                B.lars(ETA, False, step == 0)
                torch.cuda.synchronize()
                trust = _np(B.trust[0])
                assert trust[0] == 1.0 and trust[1] == 0.0, trust[:2]
                for r in range(W):
                    assert np.array_equal(_np(B.trust[r]).view(np.int32), trust.view(np.int32))
                want = _lars_want(B, [(e, g, lr, "rand") for e, g, lr in layout], trust, p, m, S, _scale(comm, None),
                                      tab, False, step == 0)
            else:
                B.sgd(0.1, 0.9, 1e-4, False, step == 0)
                want = sgd_step(p, m, S, _scale(comm, None), F32(0.1), F32(0.9), F32(1e-4), False, step == 0)
            B.check(*want, f"step {step}")
            bad = ~np.isfinite(_np(B.pv[0]))
            allowed = np.zeros(n, bool)
            allowed[[ia, ib]] = True
            assert not (bad & ~allowed).any(), np.nonzero(bad & ~allowed)[0][:8]
            assert bad[ia] and bad[ib]
            B.set_params(np.where(np.isfinite(_np(B.pv[0])), _np(B.pv[0]), F32(1.0)))   # next step from finite weights
            for r in range(W):
                mm = B.moms[r]
                mm.copy_(torch.where(torch.isfinite(mm), mm, torch.zeros_like(mm)))
    finally:
        B.free()


# ------------------------------------------------------------------------------------------------------- trainer --
def _cnn():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1, bias=False), nn.BatchNorm2d(8), nn.ReLU(),
                         nn.Conv2d(8, 16, 3, padding=1), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(),
                         nn.Linear(16, 10))


def _wrap(comm, checks):
    """Wrap both fused entry points: snapshot the bucket before the call, apply the oracle to the snapshot after it."""
    sgd, lars = comm.allreduce_sgd_window, comm.allreduce_lars_window

    def snap(grad_win, grad_off, param_win, param_off, momentum, count, kw):
        torch.cuda.synchronize()
        lw = kw.get("lowp_win")
        return (_np(grad_win.tensor(torch.float32, offset=grad_off, numel=count)),
                _np(param_win.tensor(torch.float32, offset=param_off, numel=count)), _np(momentum[:count]),
                (lambda: lw.tensor(torch.bfloat16, offset=kw["lowp_off"], numel=count)) if lw is not None else None,
                lambda: param_win.tensor(torch.float32, offset=param_off, numel=count))

    def verify(g, p, m, shadow, pnow, momentum, count, want, what):
        torch.cuda.synchronize()
        assert_bits(pnow().cpu(), _t(want[0]), f"{what}: parameters")
        assert_bits(momentum[:count].cpu(), _t(want[1]), f"{what}: momentum")
        if shadow is not None:
            assert_bits(shadow().cpu(), _t(want[2].view(np.int16)).view(torch.bfloat16), f"{what}: shadow")
        checks.append(what)

    def wrapped_sgd(grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, lr, momentum_coef=0.0,
                    weight_decay=0.0, nesterov=False, first_step=False, scale=None, **kw):
        g, p, m, shadow, pnow = snap(grad_win, grad_off, param_win, param_off, momentum, count, kw)
        if kw.get("group_map") is not None:
            lr_, mu_, wd_ = expand_groups(_np(kw["group_hyper"]), kw["group_map"].cpu().numpy(), count)
        elif getattr(comm, "_hyper", None) is not None:
            lr_, mu_, wd_ = (F32(v) for v in _np(comm._hyper))
        else:
            lr_, mu_, wd_ = F32(lr), F32(momentum_coef), F32(weight_decay)
        sgd(grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, lr, momentum_coef, weight_decay,
            nesterov, first_step, scale, **kw)
        s = _scale(comm, scale)
        verify(g, p, m, shadow, pnow, momentum, count, sgd_step(p, m, g, s, lr_, mu_, wd_, nesterov, first_step), "sgd")

    def wrapped_lars(grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, **kw):
        g, p, m, shadow, pnow = snap(grad_win, grad_off, param_win, param_off, momentum, count, kw)
        lars(grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, **kw)
        torch.cuda.synchronize()
        tab, key = _np(kw["group_hyper"]), np.repeat(kw["param_map"].cpu().numpy().astype(np.int64), 4)[:count]
        ptab = kw["param_table"].cpu().numpy().astype(np.int64)
        P = ptab.shape[0]
        trust = np.append(_np(kw["trust_out"]), F32(1.0))[key]
        grp = np.append(ptab[:, 0], 0)[key]
        s = _scale(comm, kw.get("scale"))
        gsc = (g * s).astype(F32)
        for q in range(P):                                # every LARS trust inside the oracle's interval
            sel = key == q
            if ptab[q, 1] and (gsc[sel] != 0).any() and (p[sel] != 0).any():
                lo, hi = lars_norm_interval(gsc[sel], p[sel], 1, F32(kw["trust_coefficient"]), tab[ptab[q, 0], 2])
                assert lo <= float(_np(kw["trust_out"])[q]) <= hi, q
            else:
                assert float(_np(kw["trust_out"])[q]) == 1.0, q
        want = lars_step(p, m, g, s, trust, tab[grp, 0], tab[grp, 1], tab[grp, 2], kw.get("nesterov", False),
                         kw.get("first_step", False))
        verify(g, p, m, shadow, pnow, momentum, count, want, "lars")

    comm.allreduce_sgd_window, comm.allreduce_lars_window = wrapped_sgd, wrapped_lars


@pytest.mark.parametrize("config", ["sgd", "groups", "lars", "nesterov"])
def test_trainer_launches_are_the_oracle(config):
    """DataParallelTrainer, eager, world-1 real communicator, a small channels-last CNN: every fused launch's parameters,
    momentum and bf16 shadow equal the oracle applied to the bucket as it was before the call. This pins the scale, the
    fp32 rounding of the hyper-parameters, the group and parameter maps and eta as the trainer passes them."""
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
    comm = _real_comm(f"tr-{config}")
    model = _cnn()
    no_wd = [p for p in model.parameters() if p.dim() == 1]
    kw = dict(lr=0.05, momentum=0.9, weight_decay=1e-4, cuda_graph=False, bucket_bytes=2048, bf16_params=True)
    if config == "groups":
        kw["param_groups"] = [{"params": no_wd, "weight_decay": 0.0, "lr": 0.1}]
    elif config == "lars":
        kw.update(lars=True, trust_coefficient=0.01, param_groups=[{"params": no_wd, "weight_decay": 0.0, "lars": False}])
    elif config == "nesterov":
        kw["nesterov"] = True
    tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, **kw)
    checks = []
    _wrap(comm, checks)
    g = torch.Generator().manual_seed(3)
    for _ in range(3):
        x, y = torch.randn(8, 3, 16, 16, generator=g).pin_memory(), torch.randint(0, 10, (8,), generator=g).pin_memory()
        tr.step(x, y)
    torch.cuda.synchronize()
    comm.check_error()
    assert len(checks) >= 3 * len(tr.state.buckets) and len(tr.state.buckets) > 1
    assert "lars" in checks if config == "lars" else set(checks) == {"sgd"}
    comm.destroy()


# ---------------------------------------------------------------------------------------------------------- NVLS --
@pytest.mark.multigpu
def test_nvls_steps_on_real_peers():
    """Ungrouped, grouped and LARS steps with algo="nvls" on exact-sum inputs at 2, 4 and 8 GPUs
    (tests/optimizer_mp_worker.py); skipped without multicast."""
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, here)
    from mp_launch import launch
    ran = 0
    for n in (2, 4, 8):
        if n > torch.cuda.device_count():
            continue
        rcs = launch(n, [os.path.join(here, "optimizer_mp_worker.py")], timeout=300)
        if rcs == [3] * n:
            pytest.skip("no multicast: the NVLS instantiations cannot run here")
        assert rcs == [0] * n, (n, rcs)
        ran += 1
    if not ran:
        pytest.skip("needs at least 2 GPUs")
