"""The learning-rate schedule kernel (``b200mpi_lr_schedule``) and ``DataParallelTrainer(lr_schedule=...)`` on the GPU.

Every rate the kernel writes is checked bit for bit against the exact oracle of tests/lr_schedule_oracle.py, at the step
counts of ``k_grid`` and with base rates that straddle fp32 rounding midpoints; the momentum and weight-decay columns and
guard words around every table are checked unchanged. The trainer is checked step by step in graph mode, against an
unscheduled trainer driven by ``set_lr``, and across a checkpoint."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import lr_schedule_oracle as O
from test_lr_schedule_oracle_cpu import SPECS

pytestmark = pytest.mark.gpu

GUARD = 4                   # guard elements on each side of every table
SENTINEL = -12345.5


@pytest.fixture(scope="module")
def comm():
    from mpi_operator_b200.runtime.comm import Communicator
    c = Communicator.local(1, device=0)
    yield c
    c.destroy()


def _guarded(n, dtype, fill):
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + n]


def _bases(spec, k, G, rng):
    """G base rates: the oracle's midpoint-straddling ones for m(k) first, then fixed and random ones."""
    fixed = [0.1, 1.7, 12.8, 3e-4, 0.37, 6.4]
    bs = (O.edge_bases(O.multiplier(spec, k)) + fixed)[:G] if G > 1 else [0.1]
    return bs + list(rng.uniform(1e-4, 10.0, G - len(bs)))


@pytest.mark.parametrize("G", [1, 3, 256])
@pytest.mark.parametrize("spec", SPECS, ids=[f"{s['form']}-W{s['warmup_steps']}" for s in SPECS])
def test_kernel_matches_oracle_bit_for_bit(comm, spec, G):
    from mpi_operator_b200.parallel.lr_schedule import LRSchedule
    sch = LRSchedule.from_dict(spec)
    rng = np.random.default_rng(G)
    table = torch.tensor(sch.table(), dtype=torch.float64, device="cuda")
    hbuf, hyper = _guarded(3, torch.float32, SENTINEL)
    gbuf, gflat = _guarded(3 * G, torch.float32, SENTINEL)
    sbuf, step = _guarded(1, torch.int64, -7)
    base = torch.zeros(G, dtype=torch.float64, device="cuda")
    mu_wd = torch.tensor(rng.uniform(0, 1, (G, 2)), dtype=torch.float32, device="cuda")
    for k in O.k_grid(spec):
        bases = _bases(spec, k, G, rng)
        base.copy_(torch.tensor(bases, dtype=torch.float64))
        hyper.copy_(torch.tensor([SENTINEL, 0.9, 1e-4]))
        gflat.view(G, 3)[:, 0] = SENTINEL
        gflat.view(G, 3)[:, 1:] = mu_wd
        step.fill_(k)
        before_h, before_s = hbuf.clone(), sbuf.clone()
        n0 = comm.launch_count
        comm.lr_schedule(table, sch.form, len(sch.boundaries), step, base, hyper, gflat.view(G, 3))
        torch.cuda.synchronize()
        assert comm.launch_count == n0 + 1
        want = np.array([O.rate(spec, b, k) for b in bases], dtype=np.float32)
        got_h = hyper.cpu().numpy()
        assert got_h[:1].view(np.int32) == want[:1].view(np.int32), (k, got_h[0], want[0])
        assert np.array_equal(got_h[1:], np.float32([0.9, 1e-4]))
        assert int(step) == k + 1
        for buf, old, n in ((hbuf, before_h, 3), (sbuf, before_s, 1)):
            assert torch.equal(buf[:GUARD], old[:GUARD]) and torch.equal(buf[GUARD + n:], old[GUARD + n:])
        g = gbuf.cpu().numpy()
        rows = g[GUARD:GUARD + 3 * G].reshape(G, 3)
        assert np.array_equal(rows[:, 0].view(np.int32), want.view(np.int32)), k
        assert np.array_equal(rows[:, 1:], mu_wd.cpu().numpy())
        assert np.all(g[:GUARD] == SENTINEL) and np.all(g[GUARD + 3 * G:] == SENTINEL)


def test_counter_advances_by_one_per_launch(comm):
    from mpi_operator_b200.parallel.lr_schedule import LRSchedule
    spec = SPECS[5]
    sch = LRSchedule.from_dict(spec)
    table = torch.tensor(sch.table(), dtype=torch.float64, device="cuda")
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    base = torch.tensor([0.1, 2.0, 0.37], dtype=torch.float64, device="cuda")
    hyper = torch.zeros(3, device="cuda")
    gh = torch.zeros(3, 3, device="cuda")
    for k in range(40):
        comm.lr_schedule(table, sch.form, 0, step, base, hyper, gh)
        torch.cuda.synchronize()
        assert int(step) == k + 1
        assert gh[:, 0].tolist() == [float(O.rate(spec, b, k)) for b in (0.1, 2.0, 0.37)]
    # captured in a graph, every replay advances k and writes that k's rates
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            comm.lr_schedule(table, sch.form, 0, step, base, hyper, gh, stream=torch.cuda.current_stream())
    torch.cuda.synchronize()
    assert int(step) == 40
    for k in range(40, 45):
        g.replay()
        torch.cuda.synchronize()
        assert int(step) == k + 1 and float(hyper[0]) == float(O.rate(spec, 0.1, k))


def test_entry_point_rejects_bad_arguments(comm):
    from mpi_operator_b200.runtime import _lib
    L = _lib.lib()
    t = torch.zeros(8, dtype=torch.float64, device="cuda")
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    base = torch.ones(256, dtype=torch.float64, device="cuda")
    hyper = torch.zeros(3, device="cuda")
    gh = torch.zeros(256, 3, device="cuda")
    ok = (comm._h, t.data_ptr(), 0, 0, step.data_ptr(), base.data_ptr(), 3, hyper.data_ptr(), gh.data_ptr(), None)
    bad = []
    for i in (1, 4, 5, 7):                                       # schedule, step, base, hyper
        a = list(ok)
        a[i] = None
        bad.append(a)
    for i, v in ((6, 0), (6, 257), (2, 4), (2, -1), (3, 65), (3, -1), (3, 1)):   # G; form; boundary count
        a = list(ok)
        a[i] = v
        bad.append(a)
    a = list(ok)
    a[2], a[3] = 1, 65
    bad.append(a)
    n0 = comm.launch_count
    for a in bad:
        assert L.b200mpi_lr_schedule(*a) == -1, a           # B200MPI_ERR_INVALID
    assert comm.launch_count == n0 and int(step) == 0
    gh[:, 0] = SENTINEL
    a = list(ok)
    a[8] = None                                                  # group_hyper may be NULL: only hyper is written
    assert L.b200mpi_lr_schedule(*a) == 0
    torch.cuda.synchronize()
    assert float(hyper[0]) == 1.0 and bool((gh[:, 0] == SENTINEL).all())
    assert L.b200mpi_lr_schedule(*ok) == 0
    torch.cuda.synchronize()
    assert comm.launch_count == n0 + 2 and int(step) == 2


# ---------------------------------------------------------------- trainer ----
TSCHED = {"form": "piecewise", "warmup_steps": 4, "boundaries": [6], "multipliers": [1.0, 0.1]}


def _resnet():
    from mpi_operator_b200.models import build_model
    torch.manual_seed(0)
    return build_model("resnet18", num_classes=10, width=16)


def _data(n, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(8, 3, 32, 32, generator=g).pin_memory(), torch.randint(0, 10, (8,), generator=g).pin_memory())
            for _ in range(n)]


def _groups(model, kind):
    if kind == "sgd":
        return {}
    one_d = [p for p in model.parameters() if p.dim() == 1]
    if kind == "groups":
        return {"param_groups": [{"params": one_d, "weight_decay": 0.0, "lr": 0.02}]}
    return {"lars": True, "param_groups": [{"params": one_d, "weight_decay": 0.0, "lars": False, "lr": 0.02}]}


def _trainer(comm, graph, kind="sgd", schedule=True):
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
    from mpi_operator_b200.parallel.lr_schedule import LRSchedule
    model = _resnet()
    return DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=0.05, momentum=0.9, weight_decay=1e-4,
                               cuda_graph=graph, autocast_dtype=torch.bfloat16,
                               lr_schedule=LRSchedule.from_dict(TSCHED) if schedule else None, **_groups(model, kind))


def _real_comm(tag):
    from mpi_operator_b200.runtime.comm import Communicator
    return Communicator.create(0, 1, 0, f"t-lrs-{tag}-{os.getpid()}")


@pytest.fixture
def deterministic():
    old = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = old


def _rates(bases, k):
    return [float(O.rate(TSCHED, b, k)) for b in bases]


def test_trainer_graph_mode_follows_the_schedule():
    """The capture's three eager warm-up steps use k = 0, 1, 2 (seen by every bucket launch), the captured step k = 3, and
    each replay the next k, through the end of the warm-up (k = 4) and the boundary (k = 6 / 7)."""
    comm = _real_comm("g")
    tr = _trainer(comm, graph=True, kind="groups")
    bases = [g["lr"] for g in tr.param_groups]
    seen = []
    orig = comm.allreduce_sgd_window

    def wrapped(*a, **kw):
        orig(*a, **kw)
        if not torch.cuda.is_current_stream_capturing():
            torch.cuda.synchronize()
            seen.append(tr.group_hyper[:, 0].tolist())
    comm.allreduce_sgd_window = wrapped
    data = _data(6)
    tr.step(*data[0])
    torch.cuda.synchronize()
    n = len(seen) // 3
    assert n >= 1 and len(seen) == 3 * n
    for k in range(3):
        assert all(r == _rates(bases, k) for r in seen[k * n:(k + 1) * n]), k
    assert tr.lr_schedule_step == 4 and tr.current_lrs() == _rates(bases, 3)
    for k, (x, y) in enumerate(data[1:], 4):
        tr.step(x, y)
        assert tr.lr_schedule_step == k + 1 and tr.current_lrs() == _rates(bases, k), k
    assert float(tr.hyper[0]) == _rates(bases, 8)[0]
    with_sched = tr.launches_per_step
    comm.check_error()
    comm.destroy()
    comm = _real_comm("g0")
    plain = _trainer(comm, graph=True, kind="groups", schedule=False)
    plain.step(*data[0])
    torch.cuda.synchronize()
    assert with_sched == plain.launches_per_step + 1
    comm.destroy()


@pytest.mark.parametrize("kind", ["sgd", "groups", "lars"])
def test_equivalent_to_set_lr_before_each_step(deterministic, kind):
    data = _data(8, seed=2)
    res = []
    for scheduled in (True, False):
        comm = _real_comm(f"eq{kind}{int(scheduled)}")
        tr = _trainer(comm, graph=False, kind=kind, schedule=scheduled)
        bases = [g["lr"] for g in tr.param_groups]
        for k, (x, y) in enumerate(data):
            if not scheduled:
                for g, b in enumerate(bases):
                    tr.set_lr(float(O.rate(TSCHED, b, k)), group=g)
            tr.step(x, y)
        torch.cuda.synchronize()
        res.append((tr.state.flat_param.clone(), tr._gather_shards("momentum"), tr.current_lrs()))
        comm.check_error()
        comm.destroy()
    (p0, m0, l0), (p1, m1, l1) = res
    assert l0 == l1
    assert torch.equal(p0.view(torch.int32), p1.view(torch.int32)) and torch.equal(m0.view(torch.int32), m1.view(torch.int32))


def test_resume_reproduces_the_uninterrupted_rates(deterministic):
    data = _data(7, seed=3)
    comm = _real_comm("r0")
    tr = _trainer(comm, graph=False, kind="lars")
    straight = []
    for x, y in data:
        tr.step(x, y)
        straight.append(tr.current_lrs())
    p_straight = tr.state.flat_param.clone()
    comm.destroy()
    comm = _real_comm("r1")
    tr = _trainer(comm, graph=False, kind="lars")
    for x, y in data[:3]:
        tr.step(x, y)
    sd = tr.state_dict()
    comm.destroy()
    assert sd["lr_schedule_step"] == 3
    comm = _real_comm("r2")
    tr = _trainer(comm, graph=False, kind="lars")
    tr.load_state_dict(sd)
    assert tr.current_lrs() == straight[2]
    for i, (x, y) in enumerate(data[3:], 3):
        tr.step(x, y)
        assert tr.current_lrs() == straight[i], i
    assert torch.equal(tr.state.flat_param.view(torch.int32), p_straight.view(torch.int32))
    comm.check_error()
    comm.destroy()
