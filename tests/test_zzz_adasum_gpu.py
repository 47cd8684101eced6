"""Numerics of the one-kernel Adasum allreduce (csrc/kernels/adasum.cu) against the plain PyTorch fp32 tree
(mpi_operator_b200/hvd/adasum.py: adasum_tree), on the emulated communicator (world virtual ranks on one GPU, the real
multi-rank kernel with gridDim.y == world). The file sorts last in the GPU tier on purpose: a fault in this kernel cannot
mask another test.

Reference call site: op=hvd.Adasum of examples/v2beta1/horovod/tensorflow_mnist.py:126-133 (SURVEY.md section 2.5, K6)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=[2, 4, 8])
def comm(request):
    from mpi_operator_b200.runtime.comm import Communicator
    c = Communicator.local(request.param, device=0)
    c.set_tuning(timeout_ms=5000)
    yield c
    c.destroy()


TOL = {torch.float32: (1e-4, 1e-5), torch.bfloat16: (2e-2, 2e-2), torch.float16: (2e-3, 2e-3)}


def _inputs(world, n, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn(n, device="cuda", generator=g)
    # correlated gradients (the regime Adasum is for): a shared direction plus rank noise, different norms per rank
    return [((0.5 * base + torch.randn(n, device="cuda", generator=g)) * (1.0 + 0.25 * r)).to(dtype) for r in range(world)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n", [1, 7, 1024, 4099, 65536 + 3, (1 << 20) + 5])
def test_adasum_kernel_matches_tree(comm, dtype, n):
    from mpi_operator_b200.hvd.adasum import adasum_tree
    if n * torch.empty((), dtype=dtype).element_size() > comm.adasum_max_bytes(dtype):
        pytest.skip("larger than the staging layout of the emulated communicator")
    for it in range(2):                                   # back to back: board slots and barrier words are reused
        xs = _inputs(comm.world, n, dtype, seed=n + it)
        want = adasum_tree([x.double() for x in xs]).float()      # fp64 reference: the kernel sums its dot products in fp64
        outs = [torch.empty_like(x) for x in xs] if it == 0 else xs     # out of place, then in place
        comm.adasum(xs, outs)
        torch.cuda.synchronize()
        comm.check_error()
        rtol, atol = TOL[dtype]
        for o in outs:
            torch.testing.assert_close(o.float(), want.to(dtype).float(), rtol=rtol, atol=atol)
        for o in outs[1:]:                                # identical coefficients on every rank: identical bits
            assert torch.equal(o, outs[0])


def test_adasum_kernel_identities(comm):
    """Orthogonal vectors add, identical vectors average (the two defining properties), zero vectors are neutral."""
    w, n = comm.world, 4096
    e = [torch.zeros(n, device="cuda") for _ in range(w)]
    for r in range(w):
        e[r][r::w] = 1.0
    comm.adasum(e, e)
    torch.cuda.synchronize()
    comm.check_error()
    for t in e:
        torch.testing.assert_close(t, torch.ones(n, device="cuda"))
    p = [torch.full((n,), 2.0, device="cuda") for _ in range(w)]
    comm.adasum(p, p)
    z = [torch.zeros(n, device="cuda") for _ in range(w)]
    z[0].fill_(3.0)
    comm.adasum(z, z)
    torch.cuda.synchronize()
    comm.check_error()
    for t in p:
        torch.testing.assert_close(t, torch.full((n,), 2.0, device="cuda"))
    for t in z:
        torch.testing.assert_close(t, torch.full((n,), 3.0, device="cuda"))


def test_adasum_kernel_rejects_what_it_cannot_do(comm):
    from mpi_operator_b200.runtime.comm import B200MPIError
    big = comm.adasum_max_bytes(torch.float32) // 4 + 1024
    xs = [torch.zeros(big, device="cuda") for _ in range(comm.world)]
    with pytest.raises(B200MPIError):
        comm.adasum(xs, xs)
