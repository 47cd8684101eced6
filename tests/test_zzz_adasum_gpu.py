"""The one-kernel Adasum allreduce (csrc/kernels/adasum.cu) bit for bit against the float64 oracle of
tests/adasum_oracle.py, on the emulated communicator (world virtual ranks on one GPU: the real multi-rank kernel with
gridDim.y == world) and, in the multigpu test, on real peers.

Every output must equal ``adasum_oracle.expected`` in every bit and every rank must hold the same bits. The oracle's tie
guard is given the kernel's summation depth, computed from the grid the host plans (``per`` vectors per rank, the CTA
count, the world), so a case whose answer could depend on the order of the fp64 sums fails loudly and names itself.

Covered: sizes from one element to ``adasum_max_bytes`` (sub-vector, ±1 around a vector, fewer vectors than ranks, ragged
slices, ``per`` at and around a multiple of 512 x CTAs, ~1M elements), forced CTA counts, out of place and in place back
to back, unaligned guarded buffers, input families (correlated, norms spread over 2^±40, orthogonal, identical, opposite,
zero ranks, tiny and huge scales), exact scale equivariance, NaN / ±Inf, unsupported worlds and the float64 tree.

The file sorts last in the GPU tier on purpose: a fault in this kernel cannot mask another test.
Reference call site: op=hvd.Adasum of examples/v2beta1/horovod/tensorflow_mnist.py:126-133 (SURVEY.md section 2.5, K6)."""
import contextlib
import math
import os
import sys

import pytest
import torch

from adasum_oracle import expected, kernel_depth, kernel_geometry, tree64, tree64_bound
from collective_oracle import Guarded, assert_bits, assert_ranks_agree

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
VN = {torch.float32: 4, torch.bfloat16: 8, torch.float16: 8}
NORMAL_MIN = {torch.float32: 2.0 ** -126, torch.bfloat16: 2.0 ** -126, torch.float16: 2.0 ** -14}
NORMAL_MAX = {torch.float32: 2.0 ** 127, torch.bfloat16: 2.0 ** 127, torch.float16: 2.0 ** 15}


@pytest.fixture(scope="module", params=[2, 4, 8])
def comm(request):
    from mpi_operator_b200.runtime.comm import Communicator
    c = Communicator.local(request.param, device=0)
    c.set_tuning(timeout_ms=5000)
    yield c
    c.destroy()


def emu_cap(world):
    return min(64, 132 // world)


@contextlib.contextmanager
def max_blocks(comm, n):
    old = comm.get_tuning()["max_blocks"]
    comm.set_tuning(max_blocks=n)
    try:
        yield
    finally:
        comm.set_tuning(max_blocks=old)


def want_for(comm, xs, what, info=None):
    numel, dtype = xs[0].numel(), xs[0].dtype
    _, per, blocks = kernel_geometry(numel, dtype, comm.world, max_blocks=comm.get_tuning()["max_blocks"])
    return expected(xs, dtype, depth=kernel_depth(per, blocks, comm.world, dtype), what=what, info=info)


def run_and_check(comm, xs, what, outs=None):
    """Adasum of ``xs`` into ``outs`` (default: fresh tensors, then in place); both must match the oracle bit for bit."""
    want = want_for(comm, xs, what)
    keep = [x.clone() for x in xs]
    outs = outs if outs is not None else [torch.empty_like(x) for x in xs]
    comm.adasum(xs, outs)
    torch.cuda.synchronize()
    comm.check_error()
    for r, x in enumerate(xs):
        assert torch.equal(bits(x), bits(keep[r])), f"{what}: input {r} changed"
    for r, o in enumerate(outs):
        assert_bits(o, want.to(o.device), f"{what} rank {r}")
    assert_ranks_agree(outs, what)
    comm.adasum(xs, xs)                                      # in place, back to back with the call above
    torch.cuda.synchronize()
    comm.check_error()
    for r, x in enumerate(xs):
        assert_bits(x, want.to(x.device), f"{what} in place rank {r}")
    return want


def bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


# --------------------------------------------------------------------------------------------------- inputs --
def gaussians(world, n, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn(n, device="cuda", generator=g)
    return [((0.5 * base + torch.randn(n, device="cuda", generator=g)) * (1.0 + 0.25 * r)).to(dtype) for r in range(world)]


def spread(world, n, dtype, seed):
    span = 6 if dtype == torch.float16 else 40
    g = torch.Generator().manual_seed(seed)
    ks = torch.randint(-span, span + 1, (world,), generator=g).tolist()
    return [(x.float() * 2.0 ** k).to(dtype) for x, k in zip(gaussians(world, n, torch.float32, seed), ks)]


def sizes(world, dtype):
    n = VN[dtype]
    cap = emu_cap(world)
    out = {"1": 1, "N-1": n - 1, "N+1": n + 1, "fewer-vectors-than-ranks": (world - 1) * n - 1,
           "ragged": (3 * world + 1) * n + n // 2}
    for k in (1, 2):
        p = k * 512 * cap
        out[f"per={k}*512*cta-1"] = (p - 1) * world * n
        out[f"per={k}*512*cta"] = p * world * n
        out[f"per={k}*512*cta+1"] = p * world * n + 1           # ragged: the last slice has one vector less
    return out


# ---------------------------------------------------------------------------------------------------- tests --
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [1, 7, 1024, 4099, 65536 + 3, (1 << 20) + 5])
def test_adasum_kernel_matches_tree(comm, dtype, n):
    run_and_check(comm, gaussians(comm.world, n, dtype, n), f"world {comm.world} {dtype} n={n} (seed {n})")


@pytest.mark.parametrize("dtype", DTYPES)
def test_sizes_around_vectors_slices_and_ctas(comm, dtype):
    for name, n in sizes(comm.world, dtype).items():
        run_and_check(comm, gaussians(comm.world, n, dtype, n), f"world {comm.world} {dtype} size {name} (n={n}, seed {n})")


def test_adasum_kernel_identities(comm):
    """Orthogonal vectors add, identical vectors average, a zero vector is neutral: exactly, at every rank."""
    w, n = comm.world, 4096
    e = [torch.zeros(n, device="cuda") for _ in range(w)]
    for r in range(w):
        e[r][r::w] = 1.0
    p = [torch.full((n,), 2.0, device="cuda") for _ in range(w)]
    z = [torch.zeros(n, device="cuda") for _ in range(w)]
    z[0].fill_(3.0)
    for xs, value in ((e, 1.0), (p, 2.0), (z, 3.0)):
        comm.adasum(xs, xs)
        torch.cuda.synchronize()
        comm.check_error()
        for t in xs:
            assert_bits(t, torch.full((n,), value, device="cuda"), f"identity {value}")


def test_adasum_kernel_rejects_what_it_cannot_do(comm):
    """For each dtype, the largest tensor ``adasum_max_bytes`` admits runs and matches the oracle; one element more is
    refused."""
    from mpi_operator_b200.runtime.comm import B200MPIError
    for dtype in DTYPES:
        n = comm.adasum_max_bytes(dtype) // torch.empty((), dtype=dtype).element_size()
        assert n > 0
        run_and_check(comm, gaussians(comm.world, n, dtype, 7), f"world {comm.world} {dtype} n=max={n} (seed 7)")
        xs = [torch.zeros(n + 1, device="cuda", dtype=dtype) for _ in range(comm.world)]
        with pytest.raises(B200MPIError):
            comm.adasum(xs, xs)
        del xs


@pytest.mark.parametrize("dtype", DTYPES)
def test_forced_cta_counts(comm, dtype):
    for ctas in (1, 3, emu_cap(comm.world)):
        with max_blocks(comm, ctas):
            for n in (1000, 3 * 512 * VN[dtype] * comm.world * 2 + 5):
                run_and_check(comm, gaussians(comm.world, n, dtype, ctas * 1000 + n),
                              f"world {comm.world} {dtype} ctas {ctas} n={n} (seed {ctas * 1000 + n})")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("offsets", [(1, 3), (3, 0), (0, 1)])
def test_unaligned_guarded_buffers(comm, dtype, offsets):
    oi, oo = offsets
    for n in (5, 1000, 4099 * comm.world):
        src = gaussians(comm.world, n, dtype, n)
        ins = [Guarded(n, dtype, oi, seed=10 + r) for r in range(comm.world)]
        outs = [Guarded(n, dtype, oo, seed=20 + r) for r in range(comm.world)]
        for g, x in zip(ins, src):
            g.view.copy_(x)
        for g in ins + outs:
            g.seal()
        want = want_for(comm, src, f"guarded n={n} offsets {offsets}")
        comm.adasum([g.view for g in ins], [g.view for g in outs])
        torch.cuda.synchronize()
        comm.check_error()
        for r in range(comm.world):
            assert ins[r].unchanged(), f"input {r} (offset {oi}) was written"
            assert outs[r].guards_intact(), f"output {r} (offset {oo}): bytes outside the view were written"
            assert_bits(outs[r].view, want.to("cuda"), f"guarded n={n} offsets {offsets} rank {r}")


def families(world, n, dtype):
    out = {"gaussian": gaussians(world, n, dtype, 1), "spread": spread(world, n, dtype, 2)}
    orth = [torch.zeros(n, device="cuda") for _ in range(world)]
    g = torch.Generator(device="cuda").manual_seed(3)
    vals = torch.randn(n, device="cuda", generator=g) + 3.0
    for r in range(world):
        orth[r][r::world] = vals[r::world]                         # disjoint supports: coefficients exactly 1
    out["orthogonal"] = [t.to(dtype) for t in orth]
    a = gaussians(1, n, dtype, 4)[0]
    out["identical"] = [a.clone() for _ in range(world)]
    out["opposite"] = [a.clone() if r % 2 == 0 else -a for r in range(world)]
    z = gaussians(world, n, dtype, 5)
    z[world - 1].zero_()
    out["one-zero-rank"] = z
    out["all-zero"] = [torch.zeros(n, device="cuda", dtype=dtype) for _ in range(world)]
    scales = {"2^-80": 2.0 ** -80, "1e-17": 1e-17, "2^70": 2.0 ** 70}
    if dtype == torch.float16:
        scales = {"2^-12": 2.0 ** -12, "2^12": 2.0 ** 12}
    for name, s in scales.items():
        out[f"identical-{name}"] = [torch.full((n,), s, device="cuda").to(dtype) for _ in range(world)]
        out[f"gaussian-{name}"] = [(x.float() * s).to(dtype) for x in gaussians(world, n, torch.float32, 6)]
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_input_families(comm, dtype):
    for name, xs in families(comm.world, 4099, dtype).items():
        keep = xs[0].clone()
        want = run_and_check(comm, xs, f"world {comm.world} {dtype} family {name}")
        if name.startswith("identical"):
            assert_bits(want, keep.cpu(), f"{name}: identical tensors average to themselves")
        if name == "opposite":
            assert not bool(want.float().abs().gt(0).any()), "a and -a cancel"
        if name == "all-zero":
            assert not bool(want.float().ne(0).any())


@pytest.mark.parametrize("dtype", DTYPES)
def test_scale_equivariance_is_exact(comm, dtype):
    ks = (2, 5) if dtype == torch.float16 else (-100, -60, 40, 60)   # f16: cancellations near 2^-11 must stay normal
    n = 3001
    g = torch.Generator().manual_seed(comm.world)
    xs = [(torch.sign(torch.randn(n, generator=g)) * (1 + torch.rand(n, generator=g))
           * torch.exp2(torch.randint(-4, 5, (n,), generator=g).float())).to(dtype).cuda() for _ in range(comm.world)]
    info = {}
    base = want_for(comm, xs, "unscaled", info=info)
    outs = [torch.empty_like(x) for x in xs]
    comm.adasum(xs, outs)
    torch.cuda.synchronize()
    assert_bits(outs[0], base.cuda(), "unscaled")
    for k in ks:
        assert info["min_abs"] * 2.0 ** k >= NORMAL_MIN[dtype] and info["max_abs"] * 2.0 ** k < NORMAL_MAX[dtype], \
            f"precondition: a value of the tree leaves the normal range of {dtype} at 2^{k}"
        scaled = [(x.float() * 2.0 ** k).to(dtype) for x in xs]
        comm.adasum(scaled, scaled)
        torch.cuda.synchronize()
        comm.check_error()
        for r, s in enumerate(scaled):
            assert_bits(s, (outs[0].float() * 2.0 ** k).to(dtype), f"2^{k} rank {r}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bad", [math.nan, math.inf, -math.inf])
def test_nonfinite_inputs(comm, dtype, bad):
    xs = gaussians(comm.world, 1000, dtype, 8)
    xs[comm.world - 1][17] = bad
    want = run_and_check(comm, xs, f"{bad} in the last rank")
    assert bool(torch.isnan(want.float()).all())


def test_unsupported_worlds_and_empty_tensors():
    from mpi_operator_b200.runtime.comm import B200MPIError, Communicator
    for w in (3, 6):
        c = Communicator.local(w, device=0)
        try:
            assert c.adasum_max_bytes(torch.float32) == 0
            xs = [torch.ones(64, device="cuda") for _ in range(w)]
            with pytest.raises(B200MPIError):
                c.adasum(xs, [torch.empty_like(x) for x in xs])
            before = c.launch_count
            e = [torch.empty(0, device="cuda") for _ in range(w)]
            c.adasum(e, e)
            assert c.launch_count == before
        finally:
            c.destroy()


def test_empty_tensor_launches_nothing(comm):
    before = comm.launch_count
    e = [torch.empty(0, device="cuda", dtype=torch.bfloat16) for _ in range(comm.world)]
    comm.adasum(e, e)
    assert comm.launch_count == before


@pytest.mark.parametrize("dtype", DTYPES)
def test_within_bound_of_float64_tree(comm, dtype):
    xs = gaussians(comm.world, 50000, dtype, 12)
    outs = [torch.empty_like(x) for x in xs]
    comm.adasum(xs, outs)
    torch.cuda.synchronize()
    ref, bound = tree64(xs), tree64_bound(xs, dtype)
    err = (outs[0].double().cpu() - ref).abs()
    assert bool(torch.isfinite(bound).all()) and bool((err <= bound).all()), float((err / bound).max())


@pytest.mark.multigpu
def test_adasum_on_real_peers():
    """``comm.adasum`` over 2, 4 and 8 GPUs (up to 64 CTAs per rank) against the oracle, and ``adasum_allreduce_`` with the
    kernel switch on and off (tests/adasum_mp_worker.py)."""
    sys.path.insert(0, HERE)
    from mp_launch import launch
    ran = 0
    for n in (2, 4, 8):
        if n > torch.cuda.device_count():
            continue
        for kernel in ("1", "0"):
            rcs = launch(n, [os.path.join(HERE, "adasum_mp_worker.py")], timeout=300,
                         extra_env={"B200MPI_ADASUM_KERNEL": kernel})
            assert rcs == [0] * n, (n, kernel, rcs)
        ran += 1
    assert ran > 0

