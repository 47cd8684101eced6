"""Every reducing collective entry point held bit for bit to the exact-sum oracle (tests/collective_oracle.py), at worlds 1-8.

The emulated communicator runs the real multi-rank kernels in one launch (gridDim.y == world). Inputs are chosen so that
their fp32 sum is exact in any rank order, so each output element has exactly one correct value: fp32 accumulation, the
scale applied once after the sum, one round-to-nearest-even into the tensor's dtype. Byte-moving collectives must equal the
PyTorch rearrangement bit for bit. The sizes hit less than one 16-byte vector, a partial last vector, ragged rank slices
(empty last slices at odd worlds) and payloads above the one-shot limit; a second communicator with the smallest staging
window makes every staged loop run several launches; guarded views check that no kernel writes outside its output or into
its input; NaN / Inf / fp16 overflow / subnormal inputs pin the non-finite behaviour; the fused allreduce+SGD kernel is
checked step by step against float64."""
import itertools

import pytest
import torch

from collective_oracle import Guarded, assert_bits, assert_ranks_agree, bits, exact_inputs, expected

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
OPS = [("sum", None), ("avg", None), ("max", None), ("min", None), ("sum", 0.1)]
OP_IDS = ["sum", "avg", "max", "min", "scale0.1"]
NAN, INF = float("nan"), float("inf")
PIPE_DEFAULTS = dict(min_bytes=8 << 20, chunk_bytes=1 << 20, depth=3)


@pytest.fixture(scope="module", params=list(range(1, 9)))
def comm(request):
    from mpi_operator_b200.runtime.comm import Communicator
    c = Communicator.local(request.param, device=0)
    c.set_tuning(timeout_ms=5000)
    yield c
    c.destroy()


def _esz(dtype):
    return torch.empty((), dtype=dtype).element_size()


def _nvec_elems(dtype):
    return 16 // _esz(dtype)


def _size(label, world, dtype):
    """Element counts that put the kernels on their edges."""
    N = _nvec_elems(dtype)
    return {
        "subvec": N - 1,                                   # less than one 16-byte vector
        "tail": 1000 * N + N // 2 + 1,                     # a partial last vector
        "ragged": (world + 1) * N,                         # ceil-sized rank slices; the last ones are empty at worlds >= 3
        "big": (1 << 20) // _esz(dtype) + 3 * N + 1,       # above the one-shot limit (1 MiB)
    }[label]


def _calls(comm):
    return {(o["op"], o["algo"]): o["calls"] for o in comm.stats(native_only=True)["ops"]}


def _ran(before, after):
    return {k: v - before.get(k, 0) for k, v in after.items() if v - before.get(k, 0) > 0}


def _sync(comm):
    torch.cuda.synchronize()
    comm.check_error()


def _inputs(world, n, dtype, seed):
    """Exact-sum inputs, generated on the GPU (the oracle and the comparisons run there too)."""
    return exact_inputs(world, n, dtype, seed=seed, device="cuda")


def _cuda(xs):
    """Copies handed to a collective; the originals stay for the oracle and the unchanged-input checks."""
    return [x.clone() for x in xs]


def _check_outputs(outs, want, what):
    assert_ranks_agree(outs, what)
    for r, o in enumerate(outs):
        assert_bits(o, want, f"{what} rank {r}")


# ----------------------------------------------------------------------------------------------------- allreduce --
@pytest.mark.parametrize("size", ["subvec", "tail", "ragged", "big"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("path", ["oneshot", "twoshot", "pipe"])
def test_allreduce_exact(comm, path, dtype, size):
    """sum, avg, max, min and sum with scale=0.1, out of place."""
    W = comm.world
    n = _size(size, W, dtype)
    xs0 = _inputs(W, n, dtype, seed=n + W)
    xs = _cuda(xs0)
    if path == "pipe":
        comm.set_pipe(min_bytes=0, depth=2)
    try:
        before = _calls(comm)
        for op, scale in OPS:
            outs = [torch.full_like(x, NAN) for x in xs]
            comm.allreduce(xs, outs, op=op, scale=scale, algo="oneshot" if path == "oneshot" else "twoshot")
            _sync(comm)
            _check_outputs(outs, expected(xs0, op, scale), f"allreduce {path} {op} scale={scale}")
        ran = _ran(before, _calls(comm))
    finally:
        comm.set_pipe(**PIPE_DEFAULTS)
    for x, x0 in zip(xs, xs0):
        assert torch.equal(bits(x), bits(x0)), "out-of-place allreduce changed its input"
    if path == "pipe" and W > 1:
        assert ran == {("allreduce_pipe", "twoshot"): len(OPS)}
    elif path == "oneshot" and size != "big":
        assert ran == {("allreduce", "oneshot"): len(OPS)}
    else:   # the pipe needs two ranks; the one-shot slots hold 1 MiB
        assert ran == {("allreduce", "twoshot"): len(OPS)}


@pytest.mark.parametrize("size", ["onevec", "ragged", "big"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("algo", ["oneshot", "twoshot"])
def test_allreduce_window_exact(comm, algo, dtype, size):
    W, N = comm.world, _nvec_elems(dtype)
    n = {"onevec": N, "ragged": (W + 1) * N, "big": (1 << 20) // _esz(dtype) + W * N}[size]
    off = 48
    win = comm.alloc_window(off + n * _esz(dtype) + 64)
    try:
        views = [win.tensor(dtype, rank=r, offset=off, numel=n) for r in range(W)]
        xs0 = _inputs(W, n, dtype, seed=2 * n + W)
        before = _calls(comm)
        for op, scale in OPS:
            for v, x in zip(views, xs0):
                v.copy_(x)
            comm.allreduce_window(win, off, n, dtype, op=op, scale=scale, algo=algo)
            _sync(comm)
            _check_outputs(views, expected(xs0, op, scale), f"allreduce_window {algo} {op} scale={scale}")
        used = "oneshot" if algo == "oneshot" and size != "big" else "twoshot"
        assert _ran(before, _calls(comm)) == {("allreduce", used): len(OPS)}
    finally:
        win.free()


# ------------------------------------------------------------------------------------------------ reduce-scatter --
@pytest.mark.parametrize("size", ["subvec", "tail"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("path", ["staged", "pipe", "window", "window_inplace"])
def test_reduce_scatter_exact(comm, path, dtype, size):
    W, N = comm.world, _nvec_elems(dtype)
    n = _size(size, W, dtype)
    if path.startswith("window"):
        n = -(-n // N) * N      # the window form works on whole vectors
    xs0 = _inputs(W, W * n, dtype, seed=3 * n + W)
    before = _calls(comm)
    if path.startswith("window"):
        off = 32
        win = comm.alloc_window(off + W * n * _esz(dtype))
        try:
            views = [win.tensor(dtype, rank=r, offset=off, numel=W * n) for r in range(W)]
            for op, scale in OPS:
                want = expected(xs0, op, scale)
                for v, x in zip(views, xs0):
                    v.copy_(x)
                if path == "window":
                    outs = [torch.full((n,), NAN, device="cuda", dtype=dtype) for _ in range(W)]
                    comm.reduce_scatter_window(win, off, n, dtype, op=op, scale=scale, out=outs)
                    _sync(comm)
                    for r, v in enumerate(views):
                        assert torch.equal(bits(v), bits(xs0[r])), "out-of-place reduce_scatter_window changed its input"
                else:
                    comm.reduce_scatter_window(win, off, n, dtype, op=op, scale=scale)
                    _sync(comm)
                    outs = [v[r * n:(r + 1) * n] for r, v in enumerate(views)]
                for r, o in enumerate(outs):
                    assert_bits(o, want[r * n:(r + 1) * n], f"reduce_scatter {path} {op} scale={scale} rank {r}")
        finally:
            win.free()
        assert _ran(before, _calls(comm)) == {("reduce_scatter_sym", "twoshot"): len(OPS)}
        return
    xs = _cuda(xs0)
    if path == "pipe":
        comm.set_pipe(min_bytes=0, depth=2)
    try:
        for op, scale in OPS:
            want = expected(xs0, op, scale)
            outs = [torch.full((n,), NAN, device="cuda", dtype=dtype) for _ in range(W)]
            comm.reduce_scatter(xs, outs, op=op, scale=scale)
            _sync(comm)
            for r, o in enumerate(outs):
                assert_bits(o, want[r * n:(r + 1) * n], f"reduce_scatter {path} {op} scale={scale} rank {r}")
        ran = _ran(before, _calls(comm))
    finally:
        comm.set_pipe(**PIPE_DEFAULTS)
    for x, x0 in zip(xs, xs0):
        assert torch.equal(bits(x), bits(x0)), "reduce_scatter changed its input"
    assert ran == ({("reduce_scatter_pipe", "twoshot"): len(OPS)} if path == "pipe" and W > 1
                   else {("reduce_scatter", "auto"): len(OPS)})


# -------------------------------------------------------------------------------------------------------- reduce --
@pytest.mark.parametrize("size", ["subvec", "tail", "ragged"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_reduce_exact(comm, dtype, size):
    """Roots 0 and world-1, every op; the non-root outputs are left as they were."""
    W = comm.world
    n = _size(size, W, dtype)
    xs0 = _inputs(W, n, dtype, seed=5 * n + W)
    xs = _cuda(xs0)
    fill = _inputs(W, n, dtype, seed=7)
    before = _calls(comm)
    for root in sorted({0, W - 1}):
        for op, scale in OPS:
            outs = _cuda(fill)
            comm.reduce(xs, outs, root=root, op=op, scale=scale)
            _sync(comm)
            for r in range(W):
                if r == root:
                    assert_bits(outs[r], expected(xs0, op, scale), f"reduce root {r} {op} scale={scale}")
                else:
                    assert torch.equal(bits(outs[r]), bits(fill[r])), f"reduce wrote the output of non-root rank {r}"
    for x, x0 in zip(xs, xs0):
        assert torch.equal(bits(x), bits(x0)), "reduce changed its input"
    assert _ran(before, _calls(comm)) == {("reduce", "auto"): len(OPS) * len({0, W - 1})}


# ---------------------------------------------------------------------------------------- multi-launch staging --
# Communicator.local(w, staging_bytes=1): any small staging size is raised to the minimum, the 16 MiB one-shot region plus
# 4 MiB for the staged kernels. allreduce chunks through the whole 4 MiB region; staged_op chunks through region / slots,
# rounded down to 4 KiB (slots = world for allgather / reduce_scatter / alltoall, 1 for broadcast / reduce).
STAGED_REGION = 4 << 20


@pytest.fixture(scope="module", params=[3, 8])
def small_comm(request):
    from mpi_operator_b200.runtime.comm import Communicator
    c = Communicator.local(request.param, device=0, staging_bytes=1)
    c.set_tuning(timeout_ms=5000)
    c.set_pipe(min_bytes=1 << 60)
    yield c
    c.destroy()


def _chunk(world, slots):
    return STAGED_REGION if slots is None else (STAGED_REGION // slots) // 4096 * 4096


def _multi_n(world, slots, dtype):
    """Elements of about 2.5 staging chunks plus an odd tail."""
    return (5 * _chunk(world, slots) // 2) // _esz(dtype) + 7


def _launches(comm, fn):
    before = comm.launch_count
    fn()
    _sync(comm)
    return comm.launch_count - before


@pytest.mark.parametrize("dtype,op", [(torch.float32, "sum"), (torch.bfloat16, "avg"), (torch.float16, "max")],
                         ids=["f32-sum", "bf16-avg", "f16-max"])
def test_multichunk_allreduce(small_comm, dtype, op):
    c, W = small_comm, small_comm.world
    n = _multi_n(W, None, dtype)
    xs0 = _inputs(W, n, dtype, seed=11)
    want = expected(xs0, op)
    xs = _cuda(xs0)
    outs = [torch.full_like(x, NAN) for x in xs]
    before = _calls(c)
    assert _launches(c, lambda: c.allreduce(xs, outs, op=op, algo="twoshot")) >= 3
    assert _ran(before, _calls(c)) == {("allreduce", "twoshot"): 3}
    _check_outputs(outs, want, "multi-chunk allreduce")


def test_multichunk_allgather(small_comm):
    c, W = small_comm, small_comm.world
    n = _multi_n(W, W, torch.bfloat16)
    xs0 = _inputs(W, n, torch.bfloat16, seed=12)
    xs = _cuda(xs0)
    outs = [torch.full((W * n,), NAN, device="cuda", dtype=torch.bfloat16) for _ in range(W)]
    assert _launches(c, lambda: c.allgather(xs, outs)) >= 3
    want = torch.cat(xs0)
    for o in outs:
        assert_bits(o, want, "multi-chunk allgather")


def test_multichunk_reduce_scatter(small_comm):
    c, W = small_comm, small_comm.world
    n = _multi_n(W, W, torch.bfloat16)
    xs0 = _inputs(W, W * n, torch.bfloat16, seed=13)
    want = expected(xs0, "sum")
    xs = _cuda(xs0)
    outs = [torch.full((n,), NAN, device="cuda", dtype=torch.bfloat16) for _ in range(W)]
    assert _launches(c, lambda: c.reduce_scatter(xs, outs, op="sum")) >= 3
    for r, o in enumerate(outs):
        assert_bits(o, want[r * n:(r + 1) * n], f"multi-chunk reduce_scatter rank {r}")


def test_multichunk_alltoall(small_comm):
    c, W = small_comm, small_comm.world
    n = _multi_n(W, W, torch.float32)
    xs0 = _inputs(W, W * n, torch.float32, seed=14)
    xs = _cuda(xs0)
    outs = [torch.full((W * n,), NAN, device="cuda") for _ in range(W)]
    assert _launches(c, lambda: c.alltoall(xs, outs)) >= 3
    for r, o in enumerate(outs):
        assert_bits(o, torch.cat([xs0[s][r * n:(r + 1) * n] for s in range(W)]), f"multi-chunk alltoall rank {r}")


def test_multichunk_broadcast(small_comm):
    c, W = small_comm, small_comm.world
    n = _multi_n(W, 1, torch.bfloat16)
    root = W - 1
    xs0 = _inputs(W, n, torch.bfloat16, seed=15)
    xs = _cuda(xs0)
    assert _launches(c, lambda: c.broadcast(xs, root=root)) >= 3
    for x in xs:
        assert_bits(x, xs0[root], "multi-chunk broadcast")


def test_multichunk_reduce(small_comm):
    c, W = small_comm, small_comm.world
    n = _multi_n(W, 1, torch.float32)
    xs0 = _inputs(W, n, torch.float32, seed=16)
    want = expected(xs0, "avg")
    xs = _cuda(xs0)
    outs = [torch.full_like(x, NAN) for x in xs]
    assert _launches(c, lambda: c.reduce(xs, outs, root=1, op="avg")) >= 3
    assert_bits(outs[1], want, "multi-chunk reduce")
    for r in (0, 2):
        assert bool(torch.isnan(outs[r]).all()), f"reduce wrote the output of non-root rank {r}"


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_pipe_many_chunks_per_lane(small_comm, delta):
    """depth 2 and more than 2 * lanes * depth chunks, so every staging slot is refilled; the payload ends one vector before,
    at, or one vector after a chunk boundary."""
    c, W = small_comm, small_comm.world
    lanes = max(1, min(40, (132 // W) // 3))    # P2P lanes of an emulated communicator (pipe_plan)
    chunk_vecs = max(W, 1024 // W * W)          # 16 KiB chunks, rounded down to a multiple of the world
    nvec = (2 * lanes * 2 + 3) * chunk_vecs + delta
    n = 4 * nvec
    xs0 = _inputs(W, n, torch.float32, seed=17 + delta)
    want = expected(xs0, "avg")
    xs = _cuda(xs0)
    outs = [torch.full_like(x, NAN) for x in xs]
    c.set_pipe(min_bytes=0, chunk_bytes=16 << 10, depth=2)
    try:
        before = _calls(c)
        c.allreduce(xs, outs, op="avg", algo="twoshot")
        _sync(c)
        assert _ran(before, _calls(c)) == {("allreduce_pipe", "twoshot"): 1}
    finally:
        c.set_pipe(min_bytes=1 << 60, chunk_bytes=1 << 20, depth=3)
    _check_outputs(outs, want, "pipe")


# ------------------------------------------------------------------------------------ guard bands and alignment --
GUARD_OPS = ["allreduce:oneshot", "allreduce:twoshot", "allreduce:pipe", "allgather", "allgather:pipe", "alltoall",
             "broadcast", "broadcast:pipe", "reduce_scatter", "reduce_scatter:pipe", "reduce"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("kind", GUARD_OPS)
def test_guard_bands_and_offsets(comm, kind, dtype):
    """User pointers at element offsets 0, 1 and 3 (input and output independently) into buffers with 64 sentinel bytes
    on each side: results exact, sentinels intact, out-of-place inputs and non-root outputs untouched."""
    W = comm.world
    op, _, path = kind.partition(":")
    n = 1027 if dtype == torch.float32 else 2053      # ragged last vector in both dtypes
    n_in = W * n if op in ("alltoall", "reduce_scatter") else n
    n_out = W * n if op in ("alltoall", "allgather") else n
    before = _calls(comm)
    if path == "pipe":
        comm.set_pipe(min_bytes=0, chunk_bytes=16 << 10, depth=2)
    try:
        for k, (oi, oo) in enumerate(itertools.product((0, 1, 3), (0, 1, 3))):
            what = f"{kind} in+{oi} out+{oo}"
            xs0 = _inputs(W, n_in, dtype, seed=100 + k)
            ins = [Guarded(n_in, dtype, oi, seed=200 + r) for r in range(W)]
            for g, x in zip(ins, xs0):
                g.view.copy_(x)
            ins = [g.seal() for g in ins]
            if op == "broadcast":          # in place
                root = k % W
                comm.broadcast([g.view for g in ins], root=root)
                _sync(comm)
                for g in ins:
                    assert g.guards_intact(), f"{what}: sentinel overwritten"
                    assert_bits(g.view, xs0[root], what)
                continue
            outs = [Guarded(n_out, dtype, oo, seed=300 + r).seal() for r in range(W)]
            iv, ov = [g.view for g in ins], [g.view for g in outs]
            if op == "allreduce":
                comm.allreduce(iv, ov, op="avg", algo="oneshot" if path == "oneshot" else "twoshot")
            elif op == "allgather":
                comm.allgather(iv, ov)
            elif op == "alltoall":
                comm.alltoall(iv, ov)
            elif op == "reduce_scatter":
                comm.reduce_scatter(iv, ov, op="sum")
            else:
                root = k % W
                comm.reduce(iv, ov, root=root, op="sum")
            _sync(comm)
            for r in range(W):
                assert ins[r].unchanged(), f"{what}: rank {r}'s input changed"
                assert outs[r].guards_intact(), f"{what}: rank {r}'s output sentinels overwritten"
            if op == "allreduce":
                _check_outputs(ov, expected(xs0, "avg"), what)
            elif op == "allgather":
                for o in ov:
                    assert_bits(o, torch.cat(xs0), what)
            elif op == "alltoall":
                for r, o in enumerate(ov):
                    assert_bits(o, torch.cat([xs0[s][r * n:(r + 1) * n] for s in range(W)]), f"{what} rank {r}")
            elif op == "reduce_scatter":
                want = expected(xs0, "sum")
                for r, o in enumerate(ov):
                    assert_bits(o, want[r * n:(r + 1) * n], f"{what} rank {r}")
            else:
                assert_bits(ov[root], expected(xs0, "sum"), what)
                for r in range(W):
                    if r != root:
                        assert outs[r].unchanged(), f"{what}: non-root rank {r}'s output changed"
    finally:
        comm.set_pipe(**PIPE_DEFAULTS)
    if path == "pipe" and W > 1:
        assert {name for name, _ in _ran(before, _calls(comm))} == {f"{op}_pipe"}


# ------------------------------------------------------------------------------------- non-finite values, range --
def _allreduce(comm, path, xs, op):
    outs = [torch.empty_like(x) for x in xs]
    if path == "pipe":
        comm.set_pipe(min_bytes=0, depth=2)
    try:
        comm.allreduce(xs, outs, op=op, algo="oneshot" if path == "oneshot" else "twoshot")
        _sync(comm)
    finally:
        comm.set_pipe(**PIPE_DEFAULTS)
    return outs


def _place_specials(xs):
    """NaN / +Inf / -Inf at chosen elements of chosen ranks (element j of the first 16)."""
    W = len(xs)
    xs[0][0] = NAN                                   # NaN on the first rank only
    xs[W - 1][1] = NAN                               # NaN on the last rank only
    xs[0][2] = INF                                   # +Inf meets -Inf (+Inf alone at world 1)
    if W > 1:
        xs[W - 1][2] = -INF
    for x in xs:                                     # +Inf everywhere; -Inf everywhere; NaN everywhere
        x[3], x[4], x[5] = INF, -INF, NAN
    xs[W // 2][6] = -INF                             # one -Inf among finite values
    xs[0][7] = INF                                   # same-signed infinities on two ranks
    xs[W - 1][7] = INF
    xs[0][8] = NAN                                   # NaN and +Inf
    xs[W - 1][8] = INF
    xs[(W - 1) // 2][9] = NAN                        # NaN on a middle rank
    return xs


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("path", ["oneshot", "twoshot", "pipe"])
def test_nan_and_inf(comm, path, dtype):
    """sum / avg: NaN wherever a rank has NaN or +Inf meets -Inf, same-signed infinities stay infinite. max / min follow
    fmaxf / fminf: a NaN is ignored unless every rank has NaN there (unlike torch.max)."""
    W = comm.world
    n = 1000 * _nvec_elems(dtype) + 5
    xs0 = _place_specials(_inputs(W, n, dtype, seed=21))
    for op in ("sum", "avg", "max", "min"):
        outs = _allreduce(comm, path, _cuda(xs0), op)
        _check_outputs(outs, expected(xs0, op), f"{op} {path}")
        o = outs[0][:16].cpu().float()
        if op in ("sum", "avg"):
            assert bool(torch.isnan(o[[0, 1, 5, 9]]).all())
            assert W == 1 or bool(torch.isnan(o[[2, 8]]).all())
            assert o[3] == INF and o[4] == -INF and o[6] == -INF and o[7] == INF
        else:
            assert bool(torch.isnan(o[5]))
            assert W == 1 or not bool(torch.isnan(o[[0, 1, 9]]).any())


@pytest.mark.parametrize("path", ["oneshot", "twoshot", "pipe"])
def test_fp16_partial_sums_beyond_range(comm, path):
    """fp16 values whose partial sums exceed 65504 in some rank order while the total fits must come out finite and exact
    (fp32 accumulation in every order); a total beyond the range must come out +-Inf."""
    W = comm.world
    n = 64
    xs = [torch.full((n,), 0.5, dtype=torch.float16) for _ in range(W)]
    half = -(-W // 2)
    for j in range(W):                    # element j: the positives start at rank j, so each rotation is some order
        for r in range(W):
            xs[r][j] = 60000.0 if (r - j) % W < half else -60000.0
    for r in range(W):
        xs[r][W] = 60000.0                # total W * 60000: beyond the range from world 2 up
        xs[r][W + 1] = -60000.0
    xs = [x.cuda() for x in xs]
    for op in ("sum", "avg"):
        outs = _allreduce(comm, path, _cuda(xs), op)
        _check_outputs(outs, expected(xs, op), f"fp16 range {op} {path}")
        o = outs[0].cpu().float()
        assert bool(torch.isfinite(o[:W]).all())
        if op == "sum" and W > 1:
            assert o[W] == INF and o[W + 1] == -INF


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("path", ["oneshot", "twoshot", "pipe"])
def test_subnormals_survive(comm, path, dtype):
    """bf16 and fp32 subnormal inputs are summed, scaled and packed without being flushed to zero."""
    W = comm.world
    n = 4099
    tiny = 2.0 ** (-133 if dtype == torch.bfloat16 else -149)   # the smallest subnormal of each format
    top = 127 if dtype == torch.bfloat16 else 1 << 20
    g = torch.Generator().manual_seed(31)
    xs = []
    for _ in range(W):
        m = torch.randint(1, top, (n,), generator=g).double()
        s = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()
        xs.append((m * s * tiny).to(dtype).cuda())
    assert all(bool((x != 0).all()) for x in xs)
    for op in ("sum", "avg", "max"):
        want = expected(xs, op)
        assert bool((want != 0).any())
        outs = _allreduce(comm, path, _cuda(xs), op)
        _check_outputs(outs, want, f"subnormal {op} {path}")


# ----------------------------------------------------------------------------------------------------- fused SGD --
LR_MU_WD = [(0.1, 0.9, 1e-4), (0.05, 0.5, 1e-2), (0.2, 0.0, 0.0)]


@pytest.mark.parametrize("hyper", ["value", "device"])
@pytest.mark.parametrize("nesterov", [False, True])
@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16], ids=lambda d: str(d)[6:])
def test_fused_sgd_float64(comm, gdtype, nesterov, hyper):
    """k_allreduce_sgd, three steps: each step against a float64 step from the kernel's own previous parameters and
    momentum (so errors do not compound), momentum slices against the same reference, the bf16 shadow bit for bit, all
    ranks bitwise equal. Step 0 is a first step over a NaN-filled momentum, which must not be read. With hyper="device" the
    kernel reads {lr, momentum, weight_decay} from a device tensor (set_hyper) that changes between steps, and the by-value
    arguments are deliberately wrong."""
    W, N = comm.world, _nvec_elems(gdtype)
    n, off = N * 1013, N * 24              # 1013 vectors: ragged slices at every world; the region starts inside the windows
    tot = off + n
    gwin, pwin, lwin = comm.alloc_window(tot * _esz(gdtype)), comm.alloc_window(tot * 4), comm.alloc_window(tot * 2)
    table = torch.zeros(3, device="cuda")
    try:
        gv = [gwin.tensor(gdtype, rank=r, offset=off * _esz(gdtype), numel=n) for r in range(W)]
        pv = [pwin.tensor(torch.float32, rank=r, offset=off * 4, numel=n) for r in range(W)]
        lv = [lwin.tensor(torch.bfloat16, rank=r, offset=off * 2, numel=n) for r in range(W)]
        p0 = torch.randn(n, generator=torch.Generator().manual_seed(41))
        for v in pv:
            v.copy_(p0)
        sl = comm.slice_elems(n, gdtype)
        moms = [torch.full((sl,), NAN, device="cuda") for _ in range(W)]
        if hyper == "device":
            comm.set_hyper(table)
        s32 = torch.tensor(1.0 / W, dtype=torch.float32).double()
        eps = 2.0 ** -23
        for step, (lr, mu, wd) in enumerate(LR_MU_WD):
            gs = _inputs(W, n, gdtype, seed=50 + step)
            for v, g in zip(gv, gs):
                v.copy_(g)
            p = pv[0].cpu().double()
            m = torch.cat([x.cpu() for x in moms])[:n].double()
            first = step == 0
            lr64, mu64, wd64 = (torch.tensor(v, dtype=torch.float32).double() for v in (lr, mu, wd))
            S = torch.stack([g.double() for g in gs]).sum(0).cpu()
            if hyper == "device":
                table.copy_(torch.tensor([lr, mu, wd]))
                comm.allreduce_sgd_window(gwin, off * _esz(gdtype), pwin, off * 4, moms, n, gdtype, lr=7.0, momentum_coef=0.25,
                                          weight_decay=0.5, nesterov=nesterov, first_step=first, lowp_win=lwin, lowp_off=off * 2,
                                          algo="twoshot")
            else:
                comm.allreduce_sgd_window(gwin, off * _esz(gdtype), pwin, off * 4, moms, n, gdtype, lr=lr, momentum_coef=mu,
                                          weight_decay=wd, nesterov=nesterov, first_step=first, lowp_win=lwin,
                                          lowp_off=off * 2, algo="twoshot")
            _sync(comm)
            g = S * s32 + wd64 * p
            mag_g = (S * s32).abs() + (wd64 * p).abs()
            m_ref = g if first else mu64 * m + g
            mag_m = mag_g if first else mu64 * m.abs() + mag_g
            upd = g + mu64 * m_ref if nesterov else m_ref
            mag_u = mag_g + mu64 * mag_m if nesterov else mag_m
            p_ref = p - lr64 * upd
            m_got = torch.cat([x.cpu() for x in moms])[:n].double()
            p_got = pv[0].cpu().double()
            assert bool(((m_got - m_ref).abs() <= 4 * eps * mag_m).all()), f"step {step}: momentum"
            assert bool(((p_got - p_ref).abs() <= 4 * eps * (p.abs() + lr64 * mag_u)).all()), f"step {step}: parameters"
            assert_ranks_agree(pv, f"step {step} parameters")
            for v in lv:
                assert torch.equal(bits(v), bits(pv[0].to(torch.bfloat16))), f"step {step}: bf16 shadow"
    finally:
        comm.set_hyper(None)
        for w in (gwin, pwin, lwin):
            w.free()
