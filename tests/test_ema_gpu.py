"""The weight average of the fused SGD and LARS steps (``b200mpi_allreduce_sgd_sym_ema`` / ``b200mpi_allreduce_lars_sym_ema``)
and ``DataParallelTrainer(ema_decay=...)`` on the GPU.

The kernels run on emulated communicators (world virtual ranks in one launch) and on a world-1 real communicator. Every
element of every EMA shard is checked bit for bit against the exact oracle of tests/ema_oracle.py, applied to the updated
parameters read back from the parameter window; the parameter, momentum, bf16-shadow and trust-ratio results are checked
bitwise against the entry points without the average."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from ema_oracle import ema_step

pytestmark = pytest.mark.gpu

TABLE = [[0.5, 0.9, 1e-3], [0.05, 0.8, 1e-4]]
# (elements, group, lars): ragged parameter sizes; the region's vector count is not a multiple of any world >= 2
LAYOUT = [(4, 0, 1), (12, 1, 0), (4 * 1013, 0, 1), (4 * 1013 + 2, 1, 0), (4 * 3001, 0, 1), (4 * 37, 1, 1), (4 * 9, 0, 0)]
SENTINEL = -12345.5


def _real_comm(tag):
    from mpi_operator_b200.runtime.comm import Communicator
    return Communicator.create(0, 1, 0, f"t-ema-{tag}-{os.getpid()}")


@pytest.fixture(scope="module", params=["real1", 1, 2, 3, 4, 5, 6, 7, 8])
def comm(request):
    from mpi_operator_b200.runtime.comm import Communicator
    c = _real_comm("k") if request.param == "real1" else Communicator.local(request.param, device=0)
    c.set_tuning(timeout_ms=5000)
    yield c
    c.destroy()


def _one(comm, xs):
    return xs if comm.is_local else xs[0]


def _per_rank(comm, win, dtype, off, n):
    return [win.tensor(dtype, rank=r, offset=off, numel=n) for r in range(comm.world)] if comm.is_local \
        else [win.tensor(dtype, offset=off, numel=n)]


class Region:
    """One bucket: gradient / parameter / bf16 windows, momentum and EMA shards (each EMA shard a view into a larger buffer
    whose tail holds sentinels), the group and parameter maps and the LARS board and scratch."""

    def __init__(self, comm, off=16, tail=12, d=0.999):
        self.comm, W = comm, comm.world
        self.slots, start = [], 0
        for n, *_ in LAYOUT:
            self.slots.append((start, n))
            start += -(-n // 4) * 4
        self.n, self.off = start + tail, off
        tot = off + self.n
        self.gwin, self.pwin, self.lwin = comm.alloc_window(tot * 4), comm.alloc_window(tot * 4), comm.alloc_window(tot * 2)
        self.pv = _per_rank(comm, self.pwin, torch.float32, off * 4, self.n)
        self.gv = _per_rank(comm, self.gwin, torch.float32, off * 4, self.n)
        self.lv = _per_rank(comm, self.lwin, torch.bfloat16, off * 2, self.n)
        self.per = comm.slice_elems(self.n, torch.float32)
        self.moms = [torch.zeros(self.per, device="cuda") for _ in range(W)]
        self.ema_buf = [torch.full((self.per + 64,), SENTINEL, device="cuda") for _ in range(W)]
        self.emas = [b[:self.per] for b in self.ema_buf]
        self.sched = torch.tensor([float(np.float32(d)), 0.0], dtype=torch.float64, device="cuda")
        P = len(LAYOUT)
        pmap = torch.full((self.n // 4,), P, dtype=torch.int32)
        gmap = torch.zeros(self.n // 4, dtype=torch.uint8)
        for k, ((s, n), (_, g, _)) in enumerate(zip(self.slots, LAYOUT)):
            pmap[s // 4:(s + -(-n // 4) * 4) // 4] = k
            gmap[s // 4:(s + -(-n // 4) * 4) // 4] = g
        self.pmap, self.gmap = pmap.to(torch.uint16).cuda(), gmap.cuda()
        self.table = torch.tensor([[g, l] for _, g, l in LAYOUT], dtype=torch.uint8, device="cuda")
        self.hyper = torch.tensor(TABLE, device="cuda")
        self.board = comm.alloc_window(P * W * 8 + 16)
        nb = comm.lars_scratch_bytes(self.n, P)
        self.scratch = [torch.zeros(nb, dtype=torch.uint8, device="cuda") for _ in range(W)]
        self.trust = [torch.zeros(P, device="cuda") for _ in range(W)]

    def live(self, r):
        """Elements of rank r's shard that hold its slice of the region (the rest is past the region's end)."""
        return max(0, min(self.per, self.n - r * self.per))

    def init(self, seed):
        """Parameters spanning zero, negatives, subnormals and 2^+-60 (the bulk within 2^+-30, so that LARS's sums of squares
        stay finite); the average starts near them; dead shard elements hold sentinels."""
        gen = torch.Generator(device="cuda").manual_seed(seed)
        p0 = torch.randn(self.n, device="cuda", generator=gen)
        p0 *= torch.pow(2.0, torch.randint(-30, 31, (self.n,), device="cuda", generator=gen).float())
        p0[:8] = torch.tensor([0.0, -0.0, 1e-45, -1e-45, 3e-39, -(2.0 ** 60), 2.0 ** -60, 2.0 ** 60])
        p0[self.n - 8:] = 0
        for v in self.pv:
            v.copy_(p0)
        e0 = p0 + torch.randn(self.n, device="cuda", generator=gen) * p0.abs() * 1e-2
        for r in range(self.comm.world):
            self.emas[r].fill_(SENTINEL)
            lv = self.live(r)
            self.emas[r][:lv] = e0[r * self.per:r * self.per + lv]
        self.gen = gen

    def grads(self):
        for g in self.gv:
            g.copy_(torch.randn(self.n, device="cuda", generator=self.gen) * 1e-2)

    def full_ema(self):
        return torch.cat([self.emas[r][:self.live(r)] for r in range(self.comm.world)])

    def step(self, kind, lowp, ema=True, stream=None):
        c = self.comm
        kw = dict(ema=_one(c, self.emas), ema_sched=self.sched) if ema else {}
        lk = dict(lowp_win=self.lwin, lowp_off=self.off * 2) if lowp else {}
        args = (self.gwin, self.off * 4, self.pwin, self.off * 4, _one(c, self.moms), self.n, torch.float32)
        if kind == "lars":
            c.allreduce_lars_window(*args, group_hyper=self.hyper, param_map=self.pmap, param_table=self.table,
                                    board_win=self.board, board_off=0, scratch=_one(c, self.scratch), trust_coefficient=0.5,
                                    algo="twoshot", stream=stream, trust_out=_one(c, self.trust), **lk, **kw)
        elif kind == "grouped":
            c.allreduce_sgd_window(*args, lr=9.0, momentum_coef=9.0, weight_decay=9.0, algo="twoshot", stream=stream,
                                   group_map=self.gmap, group_hyper=self.hyper, **lk, **kw)
        else:
            c.allreduce_sgd_window(*args, lr=0.05, momentum_coef=0.9, weight_decay=1e-4, algo="twoshot", stream=stream,
                                   **lk, **kw)

    def free(self):
        for w in (self.gwin, self.pwin, self.lwin, self.board):
            w.free()


def _bits(t):
    return t.contiguous().view(torch.int32)


def _np(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("kind", ["sgd", "grouped", "lars"])
@pytest.mark.parametrize("d", [0.5, 0.999, 0.9999])
def test_kernel_matches_oracle_bit_for_bit(comm, kind, d):
    R = Region(comm, d=d)
    R.init(seed=7)
    assert all((R.n // 4) % w for w in range(2, 9))         # ragged: no world >= 2 divides the vector count
    for call in range(5):
        lowp = call % 2 == 0                                 # with and without the bf16 shadow
        R.grads()
        e_old = _np(R.full_ema())
        R.sched[1:].add_(1)                                  # k advanced on the device, as the trainer does
        R.step(kind, lowp)
        torch.cuda.synchronize()
        comm.check_error()
        p_new = _np(R.pv[0])
        want = ema_step(e_old, p_new, d, call + 1)
        got = _np(R.full_ema())
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (kind, d, call,
                                                                       int((got.view(np.int32) != want.view(np.int32)).sum()))
        for r in range(comm.world):                          # nothing written past each rank's live slice
            tail = R.ema_buf[r][R.live(r):]
            assert bool((tail == SENTINEL).all()), r
        for v in R.pv:
            assert torch.equal(_bits(v), _bits(R.pv[0]))
    R.free()


@pytest.mark.parametrize("kind", ["sgd", "grouped", "lars"])
def test_average_does_not_perturb_the_step(comm, kind):
    A, B = Region(comm), Region(comm)
    A.init(seed=3)
    B.init(seed=3)
    b_ema = [b.clone() for b in B.ema_buf]
    for call in range(3):
        A.grads()
        for x, y in zip(A.gv, B.gv):
            y.copy_(x)
        A.sched[1:].add_(1)
        A.step(kind, lowp=True, ema=True)
        B.step(kind, lowp=True, ema=False)
        torch.cuda.synchronize()
        comm.check_error()
        for x, y in zip(A.pv + A.moms + A.trust, B.pv + B.moms + B.trust):
            assert torch.equal(_bits(x), _bits(y))
        for x, y in zip(A.lv, B.lv):
            assert torch.equal(x.view(torch.int16), y.view(torch.int16))
    for b, b0 in zip(B.ema_buf, b_ema):                      # the call without the average left its buffers alone
        assert torch.equal(_bits(b), _bits(b0))
    A.free()
    B.free()


def test_graph_replay_follows_k_and_equals_eager():
    comm = _real_comm("graph")
    A, B = Region(comm), Region(comm)
    A.init(seed=5)
    B.init(seed=5)
    A.grads()
    for x, y in zip(A.gv, B.gv):
        y.copy_(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm-up outside the graph: the same step on both copies
        for R in (A, B):
            R.sched[1:].add_(1)
            R.step("grouped", lowp=True, stream=s)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        B.sched[1:].add_(1)
        B.step("grouped", lowp=True, stream=torch.cuda.current_stream())
    for _ in range(4):
        A.sched[1:].add_(1)
        A.step("grouped", lowp=True)
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip(A.pv + A.moms + A.emas, B.pv + B.moms + B.emas):
            assert torch.equal(_bits(x), _bits(y))
    assert float(A.sched[1]) == float(B.sched[1]) == 5.0
    comm.check_error()
    del graph
    A.free()
    B.free()
    comm.destroy()


def test_ema_entry_points_reject_bad_arguments():
    import ctypes as C

    from mpi_operator_b200.runtime import _lib
    from mpi_operator_b200.runtime.comm import B200MPIError
    comm = _real_comm("bad")
    R = Region(comm)
    L = _lib.lib()
    ERR_INVALID = -1
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ema, sched = C.c_void_p(R.emas[0].data_ptr()), C.c_void_p(R.sched.data_ptr())

    def sgd(gdtype=_lib.F32, e=ema, s=sched):
        return L.b200mpi_allreduce_sgd_sym_ema(comm._h, R.gwin.id, R.off * 4, R.pwin.id, R.off * 4, -1, 0,
                                               C.c_void_p(R.moms[0].data_ptr()), R.n, gdtype, 1.0, 0.1, 0.9, 0.0, 0, 0,
                                               _lib.ALGO_TWOSHOT, st, None, None, 0, e, s)

    def lars(gdtype=_lib.F32, e=ema, s=sched):
        return L.b200mpi_allreduce_lars_sym_ema(comm._h, R.gwin.id, R.off * 4, R.pwin.id, R.off * 4, -1, 0,
                                                C.c_void_p(R.moms[0].data_ptr()), R.n, gdtype, 1.0, 0, 0, _lib.ALGO_TWOSHOT,
                                                st, C.c_void_p(R.hyper.data_ptr()), 2, C.c_void_p(R.pmap.data_ptr()),
                                                C.c_void_p(R.table.data_ptr()), len(LAYOUT), R.board.id, 0,
                                                C.c_void_p(R.scratch[0].data_ptr()), R.scratch[0].numel(), 0.5, None, e, s)
    for fn in (sgd, lars):
        assert fn(e=None) == ERR_INVALID
        assert fn(s=None) == ERR_INVALID
        assert fn(gdtype=_lib.BF16) == ERR_INVALID
    R.init(seed=1)
    R.sched[1] = 1.0
    assert sgd() == 0
    torch.cuda.synchronize()
    comm.check_error()
    args = (R.gwin, R.off * 4, R.pwin, R.off * 4, R.moms[0], R.n)
    with pytest.raises(B200MPIError, match="go together"):
        comm.allreduce_sgd_window(*args, torch.float32, lr=0.1, ema=R.emas[0])
    with pytest.raises(B200MPIError, match="float32 gradients"):
        comm.allreduce_sgd_window(*args, torch.bfloat16, lr=0.1, ema=R.emas[0], ema_sched=R.sched)
    with pytest.raises(B200MPIError, match="ema must be"):
        comm.allreduce_sgd_window(*args, torch.float32, lr=0.1, ema=R.ema_buf[0], ema_sched=R.sched)
    with pytest.raises(B200MPIError, match="ema_sched"):
        comm.allreduce_sgd_window(*args, torch.float32, lr=0.1, ema=R.emas[0], ema_sched=R.sched.float())
    R.free()
    comm.destroy()


# ---------------------------------------------------------------- trainer ----
def _resnet():
    from mpi_operator_b200.models import build_model
    torch.manual_seed(0)
    return build_model("resnet18", num_classes=10, width=16)


def _data(n, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(8, 3, 32, 32, generator=g).pin_memory(), torch.randint(0, 10, (8,), generator=g).pin_memory())
            for _ in range(n)]


def _trainer(comm, graph, fused=True, ema_decay=0.99, **kw):
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
    return DataParallelTrainer(_resnet(), nn.CrossEntropyLoss(), comm, lr=0.05, momentum=0.9, weight_decay=1e-4,
                               cuda_graph=graph, fused_optimizer=fused, ema_decay=ema_decay, **kw)


@pytest.fixture
def deterministic():
    old = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = old


def _log_launches(tr):
    """Record the region of every fused launch the trainer makes; eagerly, also the EMA oracle applied to what it pushed."""
    comm, st = tr.comm, tr.state
    orig = comm.allreduce_sgd_window
    state = {"calls": [], "e": _np(st.flat_param).copy(), "eager": True}

    def wrapped(grad_win, grad_off, param_win, param_off, momentum, count, *a, **kw):
        orig(grad_win, grad_off, param_win, param_off, momentum, count, *a, **kw)
        lo = param_off // 4
        state["calls"].append((lo, count))
        if state["eager"]:
            torch.cuda.synchronize()
            k = int(kw["ema_sched"][1])
            sl = slice(lo, lo + count)
            state["e"][sl] = ema_step(state["e"][sl], _np(st.flat_param[sl]), 0.99, k)
    comm.allreduce_sgd_window = wrapped
    return state


def test_trainer_average_is_the_oracle_on_every_launch():
    """Eager steps: after every step the shards equal the oracle applied, launch by launch, to the parameters each fused
    launch pushed (a bucket may be launched more than once in a step; every launch folds its result in)."""
    comm = _real_comm("tr0")
    tr = _trainer(comm, graph=False)
    log = _log_launches(tr)
    for i, (x, y) in enumerate(_data(4)):
        tr.step(x, y)
        torch.cuda.synchronize()
        assert tr.ema_updates == i + 1
        assert np.array_equal(_np(tr._gather_ema()).view(np.int32), log["e"].view(np.int32)), i
    assert log["calls"]
    comm.check_error()
    comm.destroy()


def test_trainer_average_in_graph_mode_follows_k():
    """Graph mode: k counts the capture's three eager warm-up steps and every replay; the buckets the captured step launches
    once match the oracle on the parameter window, replay after replay."""
    comm = _real_comm("tr1")
    tr = _trainer(comm, graph=True)
    log = _log_launches(tr)
    log["eager"] = False
    data = _data(5)
    tr.step(*data[0])
    torch.cuda.synchronize()
    assert tr.ema_updates == 4 and tr._graph is not None
    n = len(log["calls"]) // 4                                  # launches per step: 3 warm-up steps and the capture
    per_step = log["calls"][-n:]
    once = [c for c in set(per_step) if per_step.count(c) == 1]
    assert once
    e = _np(tr._gather_ema()).copy()
    for i, (x, y) in enumerate(data[1:], 2):
        tr.step(x, y)
        torch.cuda.synchronize()
        assert tr.ema_updates == i + 3
        p, got = _np(tr.state.flat_param), _np(tr._gather_ema())
        for lo, count in once:
            sl = slice(lo, lo + count)
            assert np.array_equal(got[sl].view(np.int32), ema_step(e[sl], p[sl], 0.99, i + 3).view(np.int32)), (i, lo)
        e = got.copy()
    comm.check_error()
    comm.destroy()


def test_unfused_average_within_one_ulp():
    comm = _real_comm("unf")
    tr = _trainer(comm, graph=False, fused=False)
    e = _np(tr.state.flat_param).copy()
    for k, (x, y) in enumerate(_data(4), 1):
        tr.step(x, y)
        torch.cuda.synchronize()
        want = ema_step(e, _np(tr.state.flat_param), 0.99, k)
        got = _np(tr._gather_ema())
        assert np.all(np.abs(got.astype(np.float64) - want) <= np.spacing(np.abs(want)).astype(np.float64)), k
        e = want
    assert tr.ema_updates == 4
    comm.destroy()


def test_evaluate_under_ema_weights_and_training_continues_bitwise(deterministic):
    data = _data(6)
    xe, ye = _data(1, seed=9)[0]
    comm_a, comm_b = _real_comm("eva"), _real_comm("evb")
    a, b = _trainer(comm_a, graph=True), _trainer(comm_b, graph=True)
    for x, y in data[:3]:
        a.step(x, y)
        b.step(x, y)
    live = a.evaluate(xe, ye)
    with a.ema_weights():
        averaged = a.evaluate(xe, ye)
        with pytest.raises(RuntimeError):
            a.step(xe, ye)
    sd = a.state_dict()
    assert a.evaluate(xe, ye) == live                        # the eval graph reads the restored windows
    for x, y in data[3:]:
        a.step(x, y)
        b.step(x, y)
    torch.cuda.synchronize()
    assert torch.equal(_bits(a.state.flat_param), _bits(b.state.flat_param))
    assert torch.equal(a.state.flat_lowp.view(torch.int16), b.state.flat_lowp.view(torch.int16))
    assert torch.equal(_bits(a._gather_ema()), _bits(b._gather_ema()))
    comm_b.destroy()
    # a fresh trainer whose model is the checkpoint's average, with the same buffers, evaluates the same
    comm_c = _real_comm("evc")
    c = _trainer(comm_c, graph=True, ema_decay=None)
    c.load_state_dict(dict(sd, model=sd["ema"]))
    assert c.evaluate(xe, ye) == averaged
    assert averaged != live
    comm_a.destroy()
    comm_c.destroy()


def test_checkpoint_resume_is_bitwise_the_uninterrupted_run(deterministic):
    data = _data(6)
    comm_a = _real_comm("cka")
    a = _trainer(comm_a, graph=False)
    for x, y in data[:3]:
        a.step(x, y)
    sd = a.state_dict()
    comm_b = _real_comm("ckb")
    b = _trainer(comm_b, graph=False)
    b.load_state_dict(sd)
    assert b.ema_updates == 3
    for x, y in data[3:]:
        a.step(x, y)
        b.step(x, y)
    torch.cuda.synchronize()
    sa, sb = a.state_dict(), b.state_dict()
    for key in ("model", "momentum", "ema"):
        for n in sa[key]:
            assert torch.equal(_bits(sa[key][n]), _bits(sb[key][n])), (key, n)
    assert sa["ema_updates"] == sb["ema_updates"] == 6
    comm_a.destroy()
    comm_b.destroy()


def test_tf_cnn_benchmarks_moving_average_eval(tmp_path):
    import re
    import subprocess
    import sys
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = os.path.join(repo, "examples/tensorflow-benchmarks/scripts/tf_cnn_benchmarks/tf_cnn_benchmarks.py")
    cmd = [sys.executable, script, "--model=resnet18", "--batch_size=8", "--num_batches=3", "--num_warmup_batches=1",
           "--image_size=64", "--moving_average_decay=0.999", "--train_dir", str(tmp_path / "ckpt")]
    first = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd="/tmp")
    assert first.returncode == 0 and "Saved checkpoint" in first.stdout, first.stdout[-1500:] + first.stderr[-2000:]
    ev = subprocess.run(cmd + ["--eval=True"], capture_output=True, text=True, timeout=600, cwd="/tmp")
    assert ev.returncode == 0 and "Restored checkpoint" in ev.stdout, ev.stdout[-1500:] + ev.stderr[-2000:]
    assert re.search(r"Accuracy @ 1 = [0-9.]+ Accuracy @ 5 = [0-9.]+ \[24 examples\]", ev.stdout), ev.stdout[-1500:]


@pytest.mark.multigpu
def test_ema_trainer_on_real_peers():
    """The trainer with ``ema_decay`` at 2 and 4 real ranks (tests/ema_mp_worker.py): SGD and LARS, two-shot and NVLS kernels,
    ``ema_weights()`` against the oracle launch by launch and bit-identical on every rank, checkpoint round trip, graph mode."""
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, here)
    from mp_launch import launch
    ran = 0
    for n in (2, 4):
        if n > torch.cuda.device_count():
            continue
        rcs = launch(n, [os.path.join(here, "ema_mp_worker.py")], timeout=300)
        assert rcs == [0] * n, (n, rcs)
        ran += 1
    assert ran > 0
