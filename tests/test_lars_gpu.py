"""Fused allreduce + LARS (``b200mpi_allreduce_lars_sym``: k_allreduce_lars_norms + k_lars_update) and LARS in
DataParallelTrainer, on the GPU.

The kernels run on emulated communicators (world virtual ranks in one launch) and on a world-1 real communicator, and are
checked against float64 on the same inputs: trust ratios, the per-step parameter change, momentum, bitwise agreement of all
ranks, the bf16 shadow, frozen groups and bitwise equality with the grouped SGD kernel outside LARS parameters."""
import copy
import ctypes as C
import os

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

EPS = 1e-8
# {lr, momentum, weight_decay}: a LARS group, a plain group, a frozen group
TABLE = [[0.5, 0.9, 1e-3], [0.05, 0.8, 1e-4], [0.0, 0.9, 1e-2]]
# (elements, group, lars, kind): one vector, a few, 1013 vectors, more vectors than one rank's slice, all-zero weights,
# a gradient that is zero on every rank, and a frozen LARS parameter
LAYOUT = [(4, 0, 1, "w"), (12, 0, 1, "w"), (4 * 1013, 0, 1, "w"), (4 * 1013 + 2, 1, 0, "w"), (4 * 3001, 0, 1, "w"),
          (4 * 50, 0, 1, "zero_w"), (4 * 20, 0, 1, "zero_g"), (4 * 37, 2, 1, "w"), (4 * 9, 1, 0, "w"), (4 * 77, 2, 0, "w")]


def _real_comm(tag):
    from mpi_operator_b200.runtime.comm import Communicator
    return Communicator.create(0, 1, 0, f"t-lars-{tag}-{os.getpid()}")


@pytest.fixture(scope="module", params=["real1", 2, 3, 4, 6, 8])
def comm(request):
    from mpi_operator_b200.runtime.comm import Communicator
    c = _real_comm("k") if request.param == "real1" else Communicator.local(request.param, device=0)
    c.set_tuning(timeout_ms=5000)
    yield c
    c.destroy()


def _per_rank(comm, win, dtype, off, n):
    return [win.tensor(dtype, rank=r, offset=off, numel=n) for r in range(comm.world)] if comm.is_local \
        else [win.tensor(dtype, offset=off, numel=n)]


def _one(comm, xs):
    return xs if comm.is_local else xs[0]


class Region:
    """Gradient / parameter / bf16 windows, momentum shards, the parameter map and table, board and scratch of one bucket."""

    def __init__(self, comm, layout, off=16, tail=12):
        self.comm, W = comm, comm.world
        self.layout = layout
        self.slots, start = [], 0
        for n, *_ in layout:
            self.slots.append((start, n))
            start += -(-n // 4) * 4
        self.n = start + tail
        self.off = off
        tot = off + self.n
        self.gwin, self.pwin, self.lwin = comm.alloc_window(tot * 4), comm.alloc_window(tot * 4), comm.alloc_window(tot * 2)
        self.pv = _per_rank(comm, self.pwin, torch.float32, off * 4, self.n)
        self.gv = _per_rank(comm, self.gwin, torch.float32, off * 4, self.n)
        self.lv = _per_rank(comm, self.lwin, torch.bfloat16, off * 2, self.n)
        self.per = comm.slice_elems(self.n, torch.float32)
        self.moms = [torch.zeros(self.per, device="cuda") for _ in range(W)]
        P = len(layout)
        pmap = torch.full((self.n // 4,), P, dtype=torch.int32)
        for k, (s, n) in enumerate(self.slots):
            pmap[s // 4:(s + -(-n // 4) * 4) // 4] = k
        self.pmap = pmap.to(torch.uint16).cuda()
        self.table = torch.tensor([[g, l] for _, g, l, _ in layout], dtype=torch.uint8, device="cuda")
        self.hyper = torch.tensor(TABLE, device="cuda")
        self.board = comm.alloc_window(P * W * 8 + 16)
        nb = comm.lars_scratch_bytes(self.n, P)
        self.scratch = [torch.zeros(nb, dtype=torch.uint8, device="cuda") for _ in range(W)]
        self.trust = [torch.zeros(P, device="cuda") for _ in range(W)]

    def group_map(self):
        gm = torch.zeros(self.n // 4, dtype=torch.uint8)
        for (s, n), (_, g, _, _) in zip(self.slots, self.layout):
            gm[s // 4:(s + -(-n // 4) * 4) // 4] = g
        return gm.cuda()

    def lars(self, nesterov=False, first_step=False, eta=0.5, stream=None, **kw):
        c = self.comm
        c.allreduce_lars_window(self.gwin, self.off * 4, self.pwin, self.off * 4, _one(c, self.moms), self.n, torch.float32,
                                group_hyper=self.hyper, param_map=self.pmap, param_table=self.table, board_win=self.board,
                                board_off=0, scratch=_one(c, self.scratch), trust_coefficient=eta, nesterov=nesterov,
                                first_step=first_step, lowp_win=self.lwin, lowp_off=self.off * 2, algo=kw.pop("algo", "twoshot"),
                                stream=stream, trust_out=_one(c, self.trust), **kw)

    def sgd(self, nesterov=False, first_step=False):
        c = self.comm
        c.allreduce_sgd_window(self.gwin, self.off * 4, self.pwin, self.off * 4, _one(c, self.moms), self.n, torch.float32,
                               lr=9.0, momentum_coef=9.0, weight_decay=9.0, nesterov=nesterov, first_step=first_step,
                               lowp_win=self.lwin, lowp_off=self.off * 2, algo="twoshot", group_map=self.group_map(),
                               group_hyper=self.hyper)

    def full_momentum(self):
        return torch.cat(self.moms)[:self.n]

    def fill(self, gen, step):
        W = self.comm.world
        if step == 0:
            p0 = torch.randn(self.n, device="cuda", generator=gen)
            for (s, n), (_, _, _, kind) in zip(self.slots, self.layout):
                if kind == "zero_w":
                    p0[s:s + n] = 0
            p0[self._pad_mask()] = 0
            for v in self.pv:
                v.copy_(p0)
        for r in range(W):
            g = torch.randn(self.n, device="cuda", generator=gen)
            for (s, n), (_, _, _, kind) in zip(self.slots, self.layout):
                if kind == "zero_g":
                    g[s:s + n] = 0
            g[self._pad_mask()] = 0
            self.gv[r].copy_(g)

    def _pad_mask(self):
        m = torch.ones(self.n, dtype=torch.bool, device="cuda")
        for s, n in self.slots:
            m[s:s + n] = False
        return m

    def reference(self, p, m, nesterov, first_step, eta):
        """float64 LARS step from (p, m): returns (p', m', trust[P])."""
        W = self.comm.world
        g = torch.stack([x.double() for x in self.gv]).sum(0) * (1.0 / W)
        p, m = p.double(), m.double()
        h = torch.tensor(TABLE, dtype=torch.float64, device="cuda")
        trust = []
        pn, mn = p.clone(), m.clone()
        for (s, n), (_, grp, lars, _) in zip(self.slots, self.layout):
            lr, mu, wd = h[grp].tolist()
            wn, gn = float(p[s:s + n].norm()), float(g[s:s + n].norm())
            t = eta * wn / (gn + wd * wn + EPS) if (lars and wn > 0 and gn > 0) else 1.0
            trust.append(t)
            d = t * (g[s:s + n] + wd * p[s:s + n])
            mj = d if first_step else mu * m[s:s + n] + d
            mn[s:s + n] = mj
            pn[s:s + n] = p[s:s + n] - lr * (d + mu * mj if nesterov else mj)
        return pn, mn, torch.tensor(trust, dtype=torch.float64)

    def free(self):
        for w in (self.gwin, self.pwin, self.lwin, self.board):
            w.free()


@pytest.mark.parametrize("nesterov", [False, True])
def test_lars_kernel_matches_float64(comm, nesterov):
    R = Region(comm, LAYOUT)
    gen = torch.Generator(device="cuda").manual_seed(11)
    frozen = torch.zeros(R.n, dtype=torch.bool, device="cuda")
    for (s, n), (_, grp, _, _) in zip(R.slots, R.layout):
        frozen[s:s + n] = grp == 2
    for m in R.moms:
        m.fill_(float("nan"))                               # first_step must not read the old momentum
    p_init = None
    for step in range(3):
        R.fill(gen, step)
        if step == 0:
            p_init = R.pv[0].clone()
        p_old = R.pv[0].clone()
        m_old = torch.zeros(R.n, device="cuda") if step == 0 else R.full_momentum().clone()
        want_p, want_m, want_t = R.reference(p_old, m_old, nesterov, step == 0, 0.5)
        R.lars(nesterov=nesterov, first_step=(step == 0))
        torch.cuda.synchronize()
        comm.check_error()
        for t in R.trust:
            torch.testing.assert_close(t.double().cpu(), want_t, rtol=1e-5, atol=0)
            assert torch.equal(t, R.trust[0])
        assert float(R.trust[0][6]) == 1.0                  # |g| = 0 on every rank
        assert (float(R.trust[0][5]) == 1.0) == (step == 0)  # |w| = 0 until its first update
        dp = (R.pv[0] - p_old).double()
        torch.testing.assert_close(dp, want_p - p_old.double(), rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(R.full_momentum().double(), want_m, rtol=1e-5, atol=1e-5)
        for v in R.pv:
            assert torch.equal(v, R.pv[0])
        for v in R.lv:
            assert torch.equal(v, R.pv[0].to(torch.bfloat16))
    assert torch.equal(R.pv[0][frozen], p_init[frozen])
    R.free()


def test_non_lars_vectors_are_bitwise_the_grouped_kernel(comm):
    A, B = Region(comm, LAYOUT), Region(comm, LAYOUT)
    gen = torch.Generator(device="cuda").manual_seed(5)
    plain = torch.zeros(A.n, dtype=torch.bool, device="cuda")
    for (s, n), (_, _, lars, _) in zip(A.slots, A.layout):
        plain[s:s + -(-n // 4) * 4] = not lars
    plain[A.slots[-1][0] + -(-A.slots[-1][1] // 4) * 4:] = True    # the bucket tail
    for step in range(3):
        A.fill(gen, step)
        for x, y in zip(A.pv + A.gv, B.pv + B.gv):
            y.copy_(x)
        A.lars(nesterov=True, first_step=(step == 0))
        B.sgd(nesterov=True, first_step=(step == 0))
        torch.cuda.synchronize()
        comm.check_error()
        for x, y in zip(A.pv + A.lv, B.pv + B.lv):
            assert torch.equal(x[plain], y[plain])
        assert torch.equal(A.full_momentum()[plain], B.full_momentum()[plain])
    A.free()
    B.free()


def test_resnet_largest_tensor_trust(comm):
    if comm.world not in (1, 8):
        pytest.skip("world 1 and 8 cover the largest tensor")
    n = 2359296                                   # 512 x 512 x 3 x 3: ResNet-50/101/152's layer4 3x3 conv
    R = Region(comm, [(n, 0, 1, "w"), (2048, 1, 0, "w")])
    gen = torch.Generator(device="cuda").manual_seed(3)
    R.fill(gen, 0)
    for v in R.pv:
        v.mul_(0.01).add_(0.003)                  # a trained-looking weight: small, not centred
    _, _, want = R.reference(R.pv[0].clone(), torch.zeros(R.n, device="cuda"), False, True, 0.001)
    R.lars(first_step=True, eta=0.001)
    torch.cuda.synchronize()
    comm.check_error()
    torch.testing.assert_close(R.trust[0].double().cpu(), want, rtol=1e-5, atol=0)
    R.free()


def test_two_calls_are_bitwise_equal(comm):
    A, B = Region(comm, LAYOUT), Region(comm, LAYOUT)
    gen = torch.Generator(device="cuda").manual_seed(9)
    for step in range(2):
        A.fill(gen, step)
        for x, y in zip(A.pv + A.gv, B.pv + B.gv):
            y.copy_(x)
        A.lars(first_step=(step == 0))
        B.lars(first_step=(step == 0))
        torch.cuda.synchronize()
        for x, y in zip(A.pv + A.lv + A.moms + A.trust, B.pv + B.lv + B.moms + B.trust):
            assert torch.equal(x, y)
    comm.check_error()
    A.free()
    B.free()


def test_graph_replay_equals_eager_and_follows_the_table():
    comm = _real_comm("graph")
    A, B = Region(comm, LAYOUT), Region(comm, LAYOUT)
    gen = torch.Generator(device="cuda").manual_seed(2)
    A.fill(gen, 0)
    for x, y in zip(A.pv + A.gv, B.pv + B.gv):
        y.copy_(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                    # warm-up outside the graph: the same step on both copies
        A.lars(stream=s)
        B.lars(stream=s)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        B.lars(stream=torch.cuda.current_stream())
    for _ in range(2):
        A.lars()
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip(A.pv + A.lv + A.moms + A.trust, B.pv + B.lv + B.moms + B.trust):
            assert torch.equal(x, y)
    B.hyper[0, 0] = 0.0                           # freeze the LARS group from the next replay on
    before = B.pv[0].clone()
    graph.replay()
    torch.cuda.synchronize()
    g0 = torch.zeros(B.n, dtype=torch.bool, device="cuda")
    for (st, n), (_, grp, _, _) in zip(B.slots, B.layout):
        g0[st:st + n] = grp == 0
    assert torch.equal(B.pv[0][g0], before[g0]) and not torch.equal(B.pv[0][~g0], before[~g0])
    comm.check_error()
    del graph
    A.free()
    B.free()
    comm.destroy()


def test_lars_entry_point_rejects_bad_arguments():
    from mpi_operator_b200.runtime import _lib
    from mpi_operator_b200.runtime.comm import B200MPIError
    comm = _real_comm("bad")
    R = Region(comm, LAYOUT)
    L = _lib.lib()
    ERR_INVALID = -1
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def raw(gdtype=_lib.F32, pmap=R.pmap, table=R.table, P=len(LAYOUT), board=R.board.id, scratch=R.scratch[0], nb=None,
            eta=0.5):
        return L.b200mpi_allreduce_lars_sym(comm._h, R.gwin.id, R.off * 4, R.pwin.id, R.off * 4, -1, 0,
                                            C.c_void_p(R.moms[0].data_ptr()), R.n, gdtype, 1.0, 0, 0, _lib.ALGO_TWOSHOT, st,
                                            C.c_void_p(R.hyper.data_ptr()), 3,
                                            C.c_void_p(pmap.data_ptr()) if pmap is not None else None,
                                            C.c_void_p(table.data_ptr()) if table is not None else None, P, board, 0,
                                            C.c_void_p(scratch.data_ptr()), scratch.numel() if nb is None else nb, eta, None)
    assert raw(gdtype=_lib.BF16) == ERR_INVALID
    assert raw(pmap=None) == ERR_INVALID and raw(table=None) == ERR_INVALID
    assert raw(P=0) == ERR_INVALID and raw(P=1025) == ERR_INVALID
    assert raw(nb=16) == ERR_INVALID
    assert raw(eta=0.0) == ERR_INVALID
    small = comm.alloc_window(len(LAYOUT) * 8 - 16)
    assert raw(board=small.id) == ERR_INVALID                  # the board needs P * world float pairs
    assert raw() == 0
    torch.cuda.synchronize()
    comm.check_error()
    kw = dict(group_hyper=R.hyper, param_map=R.pmap, param_table=R.table, board_win=R.board, board_off=0,
              scratch=R.scratch[0], trust_coefficient=0.5)
    args = (R.gwin, R.off * 4, R.pwin, R.off * 4, R.moms[0], R.n)
    with pytest.raises(B200MPIError, match="float32"):
        comm.allreduce_lars_window(*args, torch.bfloat16, **kw)
    with pytest.raises(B200MPIError, match="param_map"):
        comm.allreduce_lars_window(*args, torch.float32, **dict(kw, param_map=R.pmap[:-1]))
    with pytest.raises(B200MPIError, match="param_map"):
        comm.allreduce_lars_window(*args, torch.float32, **dict(kw, param_map=R.pmap.to(torch.int32)))
    with pytest.raises(B200MPIError, match="param_table"):
        comm.allreduce_lars_window(*args, torch.float32, **dict(kw, param_table=R.table[:, :1].contiguous()))
    with pytest.raises(B200MPIError, match="group_hyper"):
        comm.allreduce_lars_window(*args, torch.float32, **dict(kw, group_hyper=R.hyper[:, :2].contiguous()))
    with pytest.raises(B200MPIError, match="num_params"):
        big = torch.zeros(1025, 2, dtype=torch.uint8, device="cuda")
        comm.allreduce_lars_window(*args, torch.float32, **dict(kw, param_table=big))
    with pytest.raises(B200MPIError, match="board"):
        comm.allreduce_lars_window(*args, torch.float32, **dict(kw, board_win=small))
    with pytest.raises(B200MPIError, match="trust_out"):
        comm.allreduce_lars_window(*args, torch.float32, **dict(kw, trust_out=torch.zeros(3, device="cuda")))
    small.free()
    R.free()
    comm.destroy()


# ---------------------------------------------------------------- trainer ----
def _small_model():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1, bias=False), nn.BatchNorm2d(8), nn.ReLU(),
                         nn.Conv2d(8, 16, 3, padding=1), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(),
                         nn.Linear(16, 10))


def _recipe(model):
    return [{"params": [p for p in model.parameters() if p.dim() == 1], "weight_decay": 0.0, "lars": False}]


def _reference(model, data, lr, mu, wd, eta):
    """float64 LARS on the CPU, the MLPerf recipe: returns the parameters and last trust ratios by name."""
    model = copy.deepcopy(model).cpu().double()
    params = dict(model.named_parameters())
    mom = {n: torch.zeros_like(p) for n, p in params.items()}
    trust = {}
    for x, y in data:
        model.zero_grad()
        nn.functional.cross_entropy(model(x.double()), y).backward()
        with torch.no_grad():
            for n, p in params.items():
                on = p.dim() != 1
                w_ = wd if on else 0.0
                wn, gn = float(p.norm()), float(p.grad.norm())
                t = eta * wn / (gn + w_ * wn + EPS) if (on and wn > 0 and gn > 0) else 1.0
                if on:
                    trust[n] = t
                d = t * (p.grad + w_ * p)
                mom[n] = mu * mom[n] + d
                p.sub_(lr * mom[n])
    return params, trust


@pytest.mark.parametrize("graph", [False, True])
def test_trainer_fused_unfused_and_float64_agree(graph):
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        torch.manual_seed(1)
        data = [(torch.randn(8, 3, 16, 16), torch.randint(0, 10, (8,))) for _ in range(5)]
        steps = ([data[0]] * 3 + data) if graph else data        # capture warms up with 3 eager steps on the first batch
        want, want_t = _reference(_small_model(), steps, 0.5, 0.9, 1e-4, 0.01)
        got = []
        for fused in (True, False):
            comm = _real_comm(f"tr{int(graph)}{int(fused)}")
            model = _small_model()
            tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=0.5, momentum=0.9, weight_decay=1e-4,
                                     autocast_dtype=None, cuda_graph=graph, bucket_bytes=2048, fused_optimizer=fused,
                                     lars=True, trust_coefficient=0.01, param_groups=_recipe(model))
            assert len(tr.state.buckets) > 1
            for x, y in data:
                tr.step(x.pin_memory(), y.pin_memory())
            torch.cuda.synchronize()
            comm.check_error()
            got.append(({n: p.detach().double().cpu() for n, p in model.named_parameters()}, tr.lars_trust_ratios()))
            if graph and fused:
                assert tr._graph is not None
            comm.destroy()
        for params, trust in got:
            for n, p in params.items():
                torch.testing.assert_close(p, want[n].detach(), rtol=1e-5, atol=1e-5, msg=n)
            assert set(trust) == set(want_t)
            for n, t in trust.items():
                assert t == pytest.approx(want_t[n], rel=1e-4), n
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def test_resnet50_lars_in_graph_mode():
    """The MLPerf recipe on ResNet-50: one fp32 step agrees with the unfused path; with bf16, fused BN and the CUDA graph
    the loss and trust ratios are finite and set_lr between replays is honoured."""
    from mpi_operator_b200.models import build_model
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
    torch.manual_seed(1)
    x, y = torch.randn(8, 3, 64, 64).pin_memory(), torch.randint(0, 1000, (8,)).pin_memory()
    res = []
    for fused in (True, False):
        comm = _real_comm(f"r50{int(fused)}")
        torch.manual_seed(0)
        model = build_model("resnet50")
        tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=2.0, momentum=0.9, weight_decay=5e-5,
                                 autocast_dtype=None, cuda_graph=False, fused_optimizer=fused, lars=True,
                                 trust_coefficient=0.001, param_groups=_recipe(model))
        init = [m.clone() for m in tr.state.master_state().values()]
        loss = float(tr.step(x, y))
        torch.cuda.synchronize()
        comm.check_error()
        res.append((loss, {n: m - i for n, m, i in zip([n for n, _ in model.named_parameters()],
                                                        tr.state.master_state().values(), init)}, tr.lars_trust_ratios()))
        comm.destroy()
    (l0, p0, t0), (l1, p1, t1) = res
    assert l0 == pytest.approx(l1, rel=1e-6)
    assert set(t0) == set(t1) and all(t == t for t in t0.values())
    for n in t0:
        assert t0[n] == pytest.approx(t1[n], rel=1e-4), n
    for n in p0:                                   # the step taken, parameter by parameter
        assert float((p0[n] - p1[n]).norm()) <= 1e-4 * float(p1[n].norm()) + 1e-9, n

    comm = _real_comm("r50g")
    torch.manual_seed(0)
    model = build_model("resnet50")
    tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=2.0, momentum=0.9, weight_decay=5e-5,
                             autocast_dtype=torch.bfloat16, cuda_graph=True, lars=True, trust_coefficient=0.001,
                             param_groups=_recipe(model))
    for _ in range(2):
        loss = float(tr.step(x, y))
    torch.cuda.synchronize()
    comm.check_error()
    assert tr._graph is not None and loss == loss
    trust = tr.lars_trust_ratios()
    assert len(trust) == sum(p.dim() != 1 for p in model.parameters())
    assert all(0 < t < float("inf") for t in trust.values())
    before = [m.clone() for m in tr.state.master_state().values()]
    tr.set_lr(0.0)
    tr.step(x, y)
    torch.cuda.synchronize()
    after = list(tr.state.master_state().values())
    assert all(torch.equal(a, b) for a, b in zip(before, after))
    comm.check_error()
    comm.destroy()


def test_no_sync_accumulation_then_one_lars_step():
    """Accumulate one batch with no_sync, step on another: the same update as one step on the summed gradient."""
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer

    def mlp():
        torch.manual_seed(0)
        return nn.Sequential(nn.Flatten(), nn.Linear(48, 32), nn.ReLU(), nn.Linear(32, 10))
    torch.manual_seed(2)
    (x0, y0), (x1, y1) = [(torch.randn(4, 3, 4, 4), torch.randint(0, 10, (4,))) for _ in range(2)]
    kw = dict(lr=0.5, momentum=0.9, weight_decay=1e-4, autocast_dtype=None, cuda_graph=False, channels_last=False,
              lars=True, trust_coefficient=0.01)
    comm = _real_comm("ns")
    a_model = mlp()
    a = DataParallelTrainer(a_model, nn.CrossEntropyLoss(), comm, param_groups=_recipe(a_model), **kw)
    with a.no_sync():
        a.step(x0, y0)
    a.step(x1, y1)
    torch.cuda.synchronize()
    pa = {n: p.detach().clone() for n, p in a_model.named_parameters()}
    ta = a.lars_trust_ratios()
    comm.destroy()
    comm = _real_comm("ns2")
    b_model = mlp()
    two = lambda out, y: nn.functional.cross_entropy(out[:4], y[:4]) + nn.functional.cross_entropy(out[4:], y[4:])  # noqa: E731
    b = DataParallelTrainer(b_model, two, comm, param_groups=_recipe(b_model), **kw)
    b.step(torch.cat([x0, x1]), torch.cat([y0, y1]))
    torch.cuda.synchronize()
    for n, p in b_model.named_parameters():
        torch.testing.assert_close(p.detach(), pa[n], rtol=1e-5, atol=1e-6, msg=n)
    tb = b.lars_trust_ratios()
    for n in ta:
        assert ta[n] == pytest.approx(tb[n], rel=1e-5), n
    comm.check_error()
    comm.destroy()
