"""Numerics of every b200mpi collective kernel against a plain PyTorch fp32
reference, using the emulated communicator (world virtual ranks, ONE launch
per collective with gridDim.y == world) so a single GPU exercises the real
multi-rank kernels.  SURVEY.md §4 [NEW] GPU tier."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=list(range(1, 9)))
def comm(request):
    from mpi_operator_b200.runtime.comm import Communicator
    c = Communicator.local(request.param, device=0)
    c.set_tuning(timeout_ms=5000)
    yield c
    c.destroy()


def _rand(world, n, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(n, device="cuda", dtype=torch.float32, generator=g).to(dtype) for _ in range(world)]


def _ref(xs, op, scale=1.0):
    st = torch.stack([x.float() for x in xs])
    r = {"sum": st.sum(0), "avg": st.mean(0), "max": st.max(0).values, "min": st.min(0).values}[op]
    return r * scale


TOL = {torch.float32: (1e-5, 1e-5), torch.bfloat16: (2e-2, 2e-2), torch.float16: (2e-3, 2e-3)}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("algo", ["oneshot", "twoshot"])
@pytest.mark.parametrize("n", [1, 7, 1024, 4099, 65536 + 3])
@pytest.mark.parametrize("op", ["sum", "avg", "max"])
def test_allreduce_generic(comm, dtype, algo, n, op):
    xs = _rand(comm.world, n, dtype, seed=n)
    want = _ref(xs, op)
    outs = [torch.empty_like(x) for x in xs]
    comm.allreduce(xs, outs, op=op, algo=algo)
    torch.cuda.synchronize()
    comm.check_error()
    rtol, atol = TOL[dtype]
    for o in outs:
        torch.testing.assert_close(o.float(), want.to(dtype).float(), rtol=rtol, atol=atol * max(1.0, comm.world / 2))
    for o in outs[1:]:  # every rank must hold bit-identical results
        assert torch.equal(o, outs[0])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("n", [5, 4099, (1 << 20) + 13, 3 * (1 << 20) + 7])
@pytest.mark.parametrize("chunk", [16 << 10, 256 << 10])
def test_allreduce_pipelined_user_pointers(comm, dtype, n, chunk):
    """k_allreduce_pipe: lanes of copy-in / reduce / copy-out CTAs chained through flags; many chunks per lane
    (slot reuse), ragged last chunk, sizes below one chunk, out of place and in place, back to back."""
    comm.set_pipe(min_bytes=0, chunk_bytes=chunk, depth=2)
    try:
        for it in range(3):
            xs = _rand(comm.world, n, dtype, seed=n + it)
            want = _ref(xs, "avg")
            outs = [torch.empty_like(x) for x in xs] if it != 1 else xs
            comm.allreduce(xs, outs, op="avg", algo="twoshot")
            torch.cuda.synchronize()
            comm.check_error()
            rtol, atol = TOL[dtype]
            for o in outs:
                torch.testing.assert_close(o.float(), want.to(dtype).float(), rtol=rtol, atol=atol)
                assert torch.equal(o, outs[0])
        if comm.world > 1:   # a single rank has nothing to pipeline: the staged kernel runs
            assert any(o["op"] == "allreduce_pipe" for o in comm.stats(native_only=True)["ops"])
    finally:
        comm.set_pipe(min_bytes=8 << 20, chunk_bytes=1 << 20, depth=3)


@pytest.mark.parametrize("n", [3, 1000, 70001, (1 << 19) + 5])
@pytest.mark.parametrize("chunk", [16 << 10, 128 << 10])
def test_pipelined_allgather_reduce_scatter_broadcast(comm, n, chunk):
    """The other ops of k_pipe on user pointers: allgather (push + copy-out), reduce_scatter (copy-in + reduce), broadcast
    (root pushes); several chunks per lane, ragged tails, odd sizes (byte-wise slow path), back to back with each other."""
    comm.set_pipe(min_bytes=0, chunk_bytes=chunk, depth=2)
    W = comm.world
    try:
        for it in range(2):
            xs = _rand(W, n, torch.bfloat16, seed=n + it)
            outs = [torch.empty(W * n, device="cuda", dtype=torch.bfloat16) for _ in range(W)]
            comm.allgather(xs, outs)
            want = torch.cat(xs)
            ins = _rand(W, W * n, torch.float32, seed=2 * n + it)
            rs = [torch.empty(n, device="cuda", dtype=torch.float32) for _ in range(W)]
            comm.reduce_scatter(ins, rs, op="sum")
            root = (it + 1) % W
            bs = _rand(W, n, torch.float32, seed=3 * n + it)
            bwant = bs[root].clone()
            comm.broadcast(bs, root=root)
            torch.cuda.synchronize()
            comm.check_error()
            for o in outs:
                assert torch.equal(o, want)
            rwant = _ref(ins, "sum")
            for r, o in enumerate(rs):
                torch.testing.assert_close(o, rwant[r * n:(r + 1) * n], rtol=1e-5, atol=1e-5 * W)
            for b in bs:
                assert torch.equal(b, bwant)
        names = {o["op"] for o in comm.stats(native_only=True)["ops"]}
        if comm.world > 1:
            assert {"allgather_pipe", "reduce_scatter_pipe", "broadcast_pipe"} <= names
    finally:
        comm.set_pipe(min_bytes=8 << 20, chunk_bytes=1 << 20, depth=3)


def test_pipelined_and_barrier_kernels_interleave(comm):
    """The pipeline keeps its own flags and counters: interleaving it with the barrier-based kernels on the same
    staging window must stay bit-exact (integer-valued data)."""
    comm.set_pipe(min_bytes=64 << 10, chunk_bytes=32 << 10, depth=2)
    try:
        g = torch.Generator().manual_seed(4)
        sizes = torch.randint(1, 200000, (40,), generator=g).tolist()
        bufs = [(b * 8).round() for b in _rand(comm.world, 200000, torch.float32, seed=11)]
        for i, n in enumerate(sizes):
            xs = [t[:n].clone() for t in bufs]
            want = torch.stack(xs).sum(0)
            comm.allreduce(xs, xs, algo="twoshot" if i % 2 else "auto")
            if i % 5 == 0:   # a push op (first action: stores into the peers' staging) right behind an allreduce
                g_in = [t[:n].clone() for t in bufs]
                g_out = [torch.empty(comm.world * n, device="cuda") for _ in range(comm.world)]
                comm.allgather(g_in, g_out)
                for o in g_out:
                    assert torch.equal(o, torch.cat(g_in)), f"allgather at iteration {i} n={n}"
            for x in xs:
                assert torch.equal(x, want), f"iteration {i} n={n}"
        torch.cuda.synchronize()
        comm.check_error()
    finally:
        comm.set_pipe(min_bytes=8 << 20, chunk_bytes=1 << 20, depth=3)


def test_allreduce_inplace_unaligned(comm):
    base = [torch.randn(1000 + 3, device="cuda") for _ in range(comm.world)]
    xs = [b[3:] for b in base]  # 12-byte offset: exercises the byte-wise slow path
    want = _ref(xs, "sum")
    comm.allreduce(xs, xs, op="sum", algo="twoshot")
    torch.cuda.synchronize()
    for x in xs:
        torch.testing.assert_close(x, want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("algo", ["oneshot", "twoshot", "auto"])
def test_allreduce_window(comm, dtype, algo):
    n = 1 << 18
    esz = torch.empty((), dtype=dtype).element_size()
    win = comm.alloc_window(n * esz + 4096)
    views = [win.tensor(dtype, rank=r, offset=4096, numel=n) for r in range(comm.world)]
    xs = _rand(comm.world, n, dtype, seed=3)
    for v, x in zip(views, xs):
        v.copy_(x)
    want = _ref(xs, "avg")
    comm.allreduce_window(win, 4096, n, dtype, op="avg", algo=algo)
    torch.cuda.synchronize()
    comm.check_error()
    rtol, atol = TOL[dtype]
    for v in views:
        torch.testing.assert_close(v.float(), want.to(dtype).float(), rtol=rtol, atol=atol)
        assert torch.equal(v, views[0])
    win.free()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_window_allgather_reduce_scatter_broadcast(comm, dtype):
    """Zero-copy forms on a symmetric window (k_allgather_sym / k_reduce_scatter_sym / k_broadcast_sym)."""
    W = comm.world
    esz = torch.empty((), dtype=dtype).element_size()
    per = 4096 + 8                       # elements per slice (16-byte multiple in both dtypes)
    off = 256
    win = comm.alloc_window(off + W * per * esz)
    views = [win.tensor(dtype, rank=r, offset=off, numel=W * per) for r in range(W)]
    # allgather: rank r owns slice r of its own copy; everything else is poison
    xs = _rand(W, per, dtype, seed=21)
    for r, v in enumerate(views):
        v.fill_(-7.0)
        v[r * per:(r + 1) * per].copy_(xs[r])
    comm.allgather_window(win, off, per * esz)
    torch.cuda.synchronize()
    comm.check_error()
    for v in views:
        assert torch.equal(v, torch.cat(xs))
    # reduce_scatter, out of place then in place
    ins = _rand(W, W * per, dtype, seed=22)
    for v, x in zip(views, ins):
        v.copy_(x)
    want = _ref(ins, "avg")
    outs = [torch.empty(per, device="cuda", dtype=dtype) for _ in range(W)]
    comm.reduce_scatter_window(win, off, per, dtype, op="avg", out=outs)
    torch.cuda.synchronize()
    rtol, atol = TOL[dtype]
    for r, o in enumerate(outs):
        torch.testing.assert_close(o.float(), want[r * per:(r + 1) * per].to(dtype).float(), rtol=rtol, atol=atol)
    comm.reduce_scatter_window(win, off, per, dtype, op="avg")
    torch.cuda.synchronize()
    for r, v in enumerate(views):
        torch.testing.assert_close(v[r * per:(r + 1) * per].float(), want[r * per:(r + 1) * per].to(dtype).float(), rtol=rtol, atol=atol)
    # broadcast from the last rank
    root = W - 1
    for r, v in enumerate(views):
        v.fill_(float(r))
    comm.broadcast_window(win, off, W * per * esz, root=root)
    torch.cuda.synchronize()
    comm.check_error()
    for v in views:
        assert torch.equal(v, torch.full_like(v, float(root)))
    win.free()


def test_back_to_back_stress(comm):
    """300 back-to-back small allreduces of random sizes must stay bit-exact
    (flag/epoch reuse, one-shot slot double-buffering; SURVEY.md §5.2)."""
    g = torch.Generator().manual_seed(1)
    sizes = torch.randint(1, 5000, (300,), generator=g).tolist()
    bufs = _rand(comm.world, 5000, torch.float32, seed=9)
    ints = [(b * 8).round() for b in bufs]  # small integers: fp32 sums are exact in any order
    for i, n in enumerate(sizes):
        xs = [t[:n].clone() for t in ints]
        want = torch.stack(xs).sum(0)
        comm.allreduce(xs, xs, algo="oneshot" if i % 3 else "twoshot")
        if i % 50 == 49:
            torch.cuda.synchronize()
        for x in xs:
            assert torch.equal(x, want), f"iteration {i} n={n}"
    torch.cuda.synchronize()
    comm.check_error()


def test_broadcast(comm):
    for root in (0, comm.world - 1):
        xs = _rand(comm.world, 10007, torch.float32, seed=root)
        want = xs[root].clone()
        comm.broadcast(xs, root=root)
        torch.cuda.synchronize()
        for x in xs:
            assert torch.equal(x, want)


def test_allgather(comm):
    n = 3001
    xs = _rand(comm.world, n, torch.bfloat16, seed=5)
    outs = [torch.empty(comm.world * n, device="cuda", dtype=torch.bfloat16) for _ in range(comm.world)]
    comm.allgather(xs, outs)
    torch.cuda.synchronize()
    want = torch.cat(xs)
    for o in outs:
        assert torch.equal(o, want)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_reduce_scatter(comm, dtype):
    n = 2048 + 4
    xs = _rand(comm.world, comm.world * n, dtype, seed=6)
    outs = [torch.empty(n, device="cuda", dtype=dtype) for _ in range(comm.world)]
    comm.reduce_scatter(xs, outs, op="sum")
    torch.cuda.synchronize()
    want = _ref(xs, "sum")
    rtol, atol = TOL[dtype]
    for r, o in enumerate(outs):
        torch.testing.assert_close(o.float(), want[r * n:(r + 1) * n].to(dtype).float(), rtol=rtol, atol=atol * comm.world)


def test_reduce_to_root(comm):
    xs = _rand(comm.world, 5000, torch.float32, seed=7)
    outs = [torch.zeros_like(x) for x in xs]
    comm.reduce(xs, outs, root=1 % comm.world, op="sum")
    torch.cuda.synchronize()
    torch.testing.assert_close(outs[1 % comm.world], _ref(xs, "sum"), rtol=1e-5, atol=1e-5)


def test_alltoall(comm):
    n = 513
    xs = _rand(comm.world, comm.world * n, torch.float32, seed=8)
    outs = [torch.empty_like(x) for x in xs]
    comm.alltoall(xs, outs)
    torch.cuda.synchronize()
    for r in range(comm.world):
        for s in range(comm.world):
            assert torch.equal(outs[r][s * n:(s + 1) * n], xs[s][r * n:(r + 1) * n])


def test_barrier_and_launch_count(comm):
    before = comm.launch_count
    comm.barrier()
    comm.barrier()
    torch.cuda.synchronize()
    assert comm.launch_count == before + 2


@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("nesterov", [False, True])
def test_fused_allreduce_sgd(comm, gdtype, nesterov):
    """Fused grad-average + SGD(momentum, wd) == torch.optim.SGD on the averaged gradient."""
    n = 8 * 1000
    W = comm.world
    gesz = torch.empty((), dtype=gdtype).element_size()
    gwin, pwin, lwin = comm.alloc_window(n * gesz), comm.alloc_window(n * 4), comm.alloc_window(n * 2)
    p0 = torch.randn(n, device="cuda")
    pv = [pwin.tensor(torch.float32, rank=r, numel=n) for r in range(W)]
    gv = [gwin.tensor(gdtype, rank=r, numel=n) for r in range(W)]
    lv = [lwin.tensor(torch.bfloat16, rank=r, numel=n) for r in range(W)]
    for v in pv:
        v.copy_(p0)
    sl = comm.slice_elems(n, gdtype)
    moms = [torch.zeros(sl, device="cuda") for _ in range(W)]
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([ref_p], lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=nesterov)
    for step in range(3):
        gs = _rand(W, n, gdtype, seed=100 + step)
        for v, g in zip(gv, gs):
            v.copy_(g)
        ref_p.grad = torch.stack([g.float() for g in gs]).mean(0)
        opt.step()
        comm.allreduce_sgd_window(gwin, 0, pwin, 0, moms, n, gdtype, lr=0.1, momentum_coef=0.9, weight_decay=1e-4,
                                  nesterov=nesterov, first_step=(step == 0), lowp_win=lwin, algo="twoshot")
        torch.cuda.synchronize()
        comm.check_error()
        for v in pv:
            torch.testing.assert_close(v, ref_p.data, rtol=1e-5, atol=1e-5)
            assert torch.equal(v, pv[0])
        for v in lv:
            assert torch.equal(v, pv[0].to(torch.bfloat16))
    for w in (gwin, pwin, lwin):
        w.free()


def test_scale_cast():
    from mpi_operator_b200.runtime.comm import scale_cast
    x = torch.randn(10001, device="cuda")
    y = torch.empty(10001, device="cuda", dtype=torch.bfloat16)
    scale_cast(x, y, 0.5)
    torch.cuda.synchronize()
    assert torch.equal(y, (x * 0.5).to(torch.bfloat16))


@pytest.mark.parametrize("n", [300007, 1 << 20])
def test_allreduce_staged_many_blocks(comm, n):
    """Regression: copy-in / reduce / copy-out phases must share one CTA->index map."""
    xs = _rand(comm.world, n, torch.bfloat16, seed=n)
    want = _ref(xs, "sum").to(torch.bfloat16)
    comm.allreduce(xs, xs, op="sum", algo="twoshot")
    torch.cuda.synchronize()
    comm.check_error()
    for x in xs:
        torch.testing.assert_close(x.float(), want.float(), rtol=2e-2, atol=2e-2 * comm.world)
        assert torch.equal(x, xs[0])
