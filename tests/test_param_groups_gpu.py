"""Grouped fused allreduce+SGD (``b200mpi_allreduce_sgd_sym_groups``) and DataParallelTrainer parameter groups on the GPU.

The kernel runs on the emulated communicator (world virtual ranks in one launch) and on a world-1 real communicator, and is
checked against an fp32 PyTorch reference that applies each element's group hyper-parameters."""
import copy
import ctypes as C
import os

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

LR_MU_WD = [[0.1, 0.9, 1e-4], [0.02, 0.5, 0.0], [0.0, 0.9, 1e-2], [0.3, 0.0, 5e-5], [0.05, 0.99, 1e-3]]


def _real_comm(tag):
    from mpi_operator_b200.runtime.comm import Communicator
    return Communicator.create(0, 1, 0, f"t-groups-{tag}-{os.getpid()}")


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


def _region(comm, n, off_elems):
    """Gradient / parameter / bf16 windows with a region of n elements starting off_elems into them."""
    W = comm.world
    tot = off_elems + n
    gwin, pwin, lwin = comm.alloc_window(tot * 4), comm.alloc_window(tot * 4), comm.alloc_window(tot * 2)
    pv = _per_rank(comm, pwin, torch.float32, off_elems * 4, n)
    gv = _per_rank(comm, gwin, torch.float32, off_elems * 4, n)
    lv = _per_rank(comm, lwin, torch.bfloat16, off_elems * 2, n)
    sl = comm.slice_elems(n, torch.float32)
    moms = [torch.zeros(sl, device="cuda") for _ in range(W)]
    return (gwin, pwin, lwin), pv, gv, lv, moms


def _call(comm, wins, moms, n, off_elems, **kw):
    gwin, pwin, lwin = wins
    comm.allreduce_sgd_window(gwin, off_elems * 4, pwin, off_elems * 4, moms if comm.is_local else moms[0], n, torch.float32,
                              lowp_win=lwin, lowp_off=off_elems * 2, algo=kw.pop("algo", "twoshot"), **kw)


@pytest.mark.parametrize("nesterov", [False, True])
def test_grouped_kernel_matches_per_element_reference(comm, nesterov):
    W = comm.world
    n, off = 4 * 1013, 4 * 24           # 1013 vectors: ragged slices at every world size; the region starts inside the window
    wins, pv, gv, lv, moms = _region(comm, n, off)
    gen = torch.Generator(device="cuda").manual_seed(7)
    p0 = torch.randn(n, device="cuda", generator=gen)
    for v in pv:
        v.copy_(p0)
    table = torch.tensor(LR_MU_WD, device="cuda")
    gmap = torch.randint(0, len(LR_MU_WD), (n // 4,), device="cuda", generator=gen).to(torch.uint8)
    assert len(set(gmap.tolist())) >= 3
    h = table[gmap.long()].repeat_interleave(4, dim=0)      # per-element {lr, mu, wd}
    lr, mu, wd = h[:, 0], h[:, 1], h[:, 2]
    ref_p, ref_m = p0.clone(), None
    for m in moms:
        m.fill_(float("nan"))                               # first_step must not read the old momentum
    for step in range(3):
        gs = [torch.randn(n, device="cuda", generator=gen) for _ in range(W)]
        for v, g in zip(gv, gs):
            v.copy_(g)
        g = torch.stack(gs).sum(0) * (1.0 / W) + wd * ref_p
        ref_m = g if step == 0 else mu * ref_m + g
        ref_p = ref_p - lr * (g + mu * ref_m if nesterov else ref_m)
        _call(comm, wins, moms, n, off, lr=9.0, momentum_coef=9.0, weight_decay=9.0, nesterov=nesterov,
              first_step=(step == 0), group_map=gmap, group_hyper=table)
        torch.cuda.synchronize()
        comm.check_error()
        for v in pv:
            torch.testing.assert_close(v, ref_p, rtol=1e-5, atol=1e-5)
            assert torch.equal(v, pv[0])                    # every rank holds the same bits
        for v in lv:
            assert torch.equal(v, pv[0].to(torch.bfloat16))
    frozen = (gmap == 2).repeat_interleave(4)               # lr 0: exactly the initial values
    assert torch.equal(pv[0][frozen], p0[frozen])
    for w in wins:
        w.free()


def test_one_group_is_bitwise_the_ungrouped_kernel(comm):
    n, off = 4 * 777, 8
    lr, mu, wd = 0.07, 0.9, 3e-4
    a = _region(comm, n, off)
    b = _region(comm, n, off)
    gen = torch.Generator(device="cuda").manual_seed(3)
    p0 = torch.randn(n, device="cuda", generator=gen)
    for v in a[1] + b[1]:
        v.copy_(p0)
    table = torch.tensor([[lr, mu, wd]], device="cuda")
    gmap = torch.zeros(n // 4, dtype=torch.uint8, device="cuda")
    for step in range(3):
        for r in range(len(a[2])):
            g = torch.randn(n, device="cuda", generator=gen)
            a[2][r].copy_(g)
            b[2][r].copy_(g)
        _call(comm, a[0], a[4], n, off, lr=lr, momentum_coef=mu, weight_decay=wd, nesterov=True, first_step=(step == 0))
        _call(comm, b[0], b[4], n, off, lr=lr, momentum_coef=mu, weight_decay=wd, nesterov=True, first_step=(step == 0),
              group_map=gmap, group_hyper=table)
        torch.cuda.synchronize()
        comm.check_error()
        for x, y in zip(a[1] + a[3] + a[4], b[1] + b[3] + b[4]):   # parameters, bf16 shadow, momentum
            assert torch.equal(x, y)
    for w in a[0] + b[0]:
        w.free()


def test_nvls_grouped_kernel_where_multicast_exists(comm):
    if not comm.has_multicast:
        pytest.skip("no NVLS multicast on this communicator")
    n = 4 * 4096
    wins, pv, gv, lv, moms = _region(comm, n, 0)
    p0 = torch.randn(n, device="cuda")
    for v in pv:
        v.copy_(p0)
    table = torch.tensor(LR_MU_WD, device="cuda")
    gmap = (torch.arange(n // 4, device="cuda") % len(LR_MU_WD)).to(torch.uint8)
    gs = [torch.randn(n, device="cuda") for _ in range(comm.world)]
    for v, g in zip(gv, gs):
        v.copy_(g)
    h = table[gmap.long()].repeat_interleave(4, dim=0)
    want = p0 - h[:, 0] * (torch.stack(gs).mean(0) + h[:, 2] * p0)
    _call(comm, wins, moms, n, 0, lr=1.0, first_step=True, group_map=gmap, group_hyper=table, algo="nvls")
    torch.cuda.synchronize()
    comm.check_error()
    for v in pv:
        torch.testing.assert_close(v, want, rtol=1e-5, atol=1e-5)
    for w in wins:
        w.free()


def test_table_changes_between_graph_replays_take_effect():
    comm = _real_comm("graph")
    n = 4 * 512
    wins, pv, gv, lv, moms = _region(comm, n, 0)
    p0 = torch.randn(n, device="cuda")
    pv[0].copy_(p0)
    gv[0].copy_(torch.randn(n, device="cuda"))
    table = torch.tensor([[0.1, 0.0, 0.0], [0.1, 0.0, 0.0]], device="cuda")
    gmap = (torch.arange(n // 4, device="cuda") % 2).to(torch.uint8)
    one = gmap.repeat_interleave(4) == 1
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _call(comm, wins, moms, n, 0, lr=0.0, group_map=gmap, group_hyper=table, stream=s)   # warm-up, outside the graph
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _call(comm, wins, moms, n, 0, lr=0.0, group_map=gmap, group_hyper=table, stream=torch.cuda.current_stream())
    g = gv[0].clone()
    before = pv[0].clone()
    graph.replay()
    torch.cuda.synchronize()
    torch.testing.assert_close(pv[0], before - 0.1 * g, rtol=1e-6, atol=1e-6)
    table[1, 0] = 0.0                                       # freeze group 1 from the next replay on
    before = pv[0].clone()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(pv[0][one], before[one])
    torch.testing.assert_close(pv[0][~one], (before - 0.1 * g)[~one], rtol=1e-6, atol=1e-6)
    table[1] = torch.tensor([0.5, 0.0, 0.0])
    before = pv[0].clone()
    graph.replay()
    torch.cuda.synchronize()
    torch.testing.assert_close(pv[0][one], (before - 0.5 * g)[one], rtol=1e-6, atol=1e-6)
    comm.check_error()
    del graph
    for w in wins:
        w.free()
    comm.destroy()


def test_grouped_entry_point_rejects_bad_arguments():
    from mpi_operator_b200.runtime import _lib
    from mpi_operator_b200.runtime.comm import B200MPIError
    comm = _real_comm("bad")
    n = 4 * 64
    (gwin, pwin, lwin), pv, gv, lv, moms = _region(comm, n, 0)
    table = torch.zeros(3, 3, device="cuda")
    gmap = torch.zeros(n // 4, dtype=torch.uint8, device="cuda")
    L = _lib.lib()
    ERR_INVALID = -1

    def raw(gdtype, gm, gh, ng):
        return L.b200mpi_allreduce_sgd_sym_groups(comm._h, gwin.id, 0, pwin.id, 0, -1, 0, C.c_void_p(moms[0].data_ptr()), n,
                                                  gdtype, 1.0, 0.1, 0.9, 0.0, 0, 0, _lib.ALGO_TWOSHOT,
                                                  C.c_void_p(torch.cuda.current_stream().cuda_stream), gm, gh, ng)
    m, h = C.c_void_p(gmap.data_ptr()), C.c_void_p(table.data_ptr())
    assert raw(_lib.BF16, m, h, 3) == ERR_INVALID
    assert raw(_lib.F16, m, h, 3) == ERR_INVALID
    assert raw(_lib.F32, m, h, 0) == ERR_INVALID
    assert raw(_lib.F32, m, h, 257) == ERR_INVALID
    assert raw(_lib.F32, m, None, 3) == ERR_INVALID
    assert raw(_lib.F32, None, h, 3) == ERR_INVALID
    assert raw(_lib.F32, m, h, 3) == 0
    assert raw(_lib.F32, None, None, 0) == 0                 # no groups: the ungrouped step
    torch.cuda.synchronize()
    comm.check_error()
    with pytest.raises(B200MPIError, match="float32"):
        comm.allreduce_sgd_window(gwin, 0, pwin, 0, moms[0], n, torch.bfloat16, lr=0.1, group_map=gmap, group_hyper=table)
    with pytest.raises(B200MPIError, match="together"):
        comm.allreduce_sgd_window(gwin, 0, pwin, 0, moms[0], n, torch.float32, lr=0.1, group_map=gmap)
    with pytest.raises(B200MPIError, match="group_map"):
        comm.allreduce_sgd_window(gwin, 0, pwin, 0, moms[0], n, torch.float32, lr=0.1, group_map=gmap[:-1], group_hyper=table)
    with pytest.raises(B200MPIError, match="group_map"):
        comm.allreduce_sgd_window(gwin, 0, pwin, 0, moms[0], n, torch.float32, lr=0.1, group_map=gmap.cpu(), group_hyper=table)
    with pytest.raises(B200MPIError, match="group_hyper"):
        comm.allreduce_sgd_window(gwin, 0, pwin, 0, moms[0], n, torch.float32, lr=0.1, group_map=gmap, group_hyper=table[:, :2])
    for w in (gwin, pwin, lwin):
        w.free()
    comm.destroy()


# ---------------------------------------------------------------- trainer ----
def _small_model():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1, bias=False), nn.BatchNorm2d(8), nn.ReLU(),
                         nn.Conv2d(8, 16, 3, padding=1), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(),
                         nn.Linear(16, 10))


def _groups(model):
    return [{"params": [p for p in model.parameters() if p.dim() == 1], "weight_decay": 0.0},
            {"params": [model[7].weight], "lr": 0.1, "momentum": 0.5}]


@pytest.mark.parametrize("graph", [False, True])
def test_trainer_with_groups_matches_torch_sgd(graph):
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
    comm = _real_comm(f"trainer{int(graph)}")
    model = _small_model()
    ref = copy.deepcopy(model).cuda().to(memory_format=torch.channels_last)
    listed = {id(p) for g in _groups(ref) for p in g["params"]}
    opt = torch.optim.SGD([{"params": [p for p in ref.parameters() if id(p) not in listed]}] + _groups(ref),
                          lr=0.05, momentum=0.9, weight_decay=1e-4)
    tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=0.05, momentum=0.9, weight_decay=1e-4,
                             autocast_dtype=None, cuda_graph=graph, bucket_bytes=2048, param_groups=_groups(model))
    assert len(tr.state.buckets) > 1
    torch.manual_seed(1)
    xs = [torch.randn(8, 3, 16, 16) for _ in range(6)]
    ys = [torch.randint(0, 10, (8,)) for _ in range(6)]
    warm = 3 if graph else 0
    for i, (x, y) in enumerate(zip(xs, ys)):
        tr.step(x.pin_memory(), y.pin_memory())
        for _ in range((warm + 1) if (graph and i == 0) else 1):
            opt.zero_grad()
            nn.functional.cross_entropy(ref(x.cuda().contiguous(memory_format=torch.channels_last)), y.cuda()).backward()
            opt.step()
    torch.cuda.synchronize()
    comm.check_error()
    for p, q in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(p.data, q.data, rtol=2e-4, atol=2e-5)
    assert tr.launches_per_step == len(tr.state.buckets)
    comm.destroy()


def test_resnet50_frozen_group_in_graph_mode():
    """bf16, fused BN and the fused 1x1 path, CUDA graph: a group at lr 0 keeps its initial bits while the rest trains, and
    set_lr(0.0, group=k) between replays freezes group k from the next replay on."""
    from mpi_operator_b200.models import build_model
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
    comm = _real_comm("r50")
    torch.manual_seed(0)
    model = build_model("resnet50")
    frozen = [p for n, p in model.named_parameters() if n.startswith("layer4")]
    head = [model.fc.weight, model.fc.bias]
    tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=0.05, momentum=0.9, weight_decay=5e-5,
                             autocast_dtype=torch.bfloat16, cuda_graph=True,
                             param_groups=[{"params": frozen, "lr": 0.0}, {"params": head}])
    masters = lambda: {n: m.clone() for n, m in zip(  # noqa: E731
        [n for n, _ in model.named_parameters()], tr.state.master_state().values())}
    init = masters()
    names = tr.param_groups
    torch.manual_seed(1)
    x, y = torch.randn(8, 3, 64, 64).pin_memory(), torch.randint(0, 1000, (8,)).pin_memory()
    for _ in range(3):
        tr.step(x, y)
    torch.cuda.synchronize()
    comm.check_error()
    assert tr._graph is not None
    now = masters()
    for n in names[1]["params"]:
        assert torch.equal(now[n], init[n]), n
    assert all(not torch.equal(now[n], init[n]) for n in names[2]["params"])
    assert sum(not torch.equal(now[n], init[n]) for n in names[0]["params"]) > len(names[0]["params"]) // 2
    tr.set_lr(0.0, group=2)
    tr.step(x, y)
    torch.cuda.synchronize()
    after = masters()
    for n in names[2]["params"]:
        assert torch.equal(after[n], now[n]), n
    for n in names[1]["params"]:
        assert torch.equal(after[n], init[n]), n
    assert sum(not torch.equal(after[n], now[n]) for n in names[0]["params"]) > len(names[0]["params"]) // 2
    st = tr.state
    assert st.flat_lowp is None or torch.equal(st.flat_lowp, st.flat_param.to(torch.bfloat16))
    comm.check_error()
    comm.destroy()
