"""Multi-process (one rank per GPU) Adasum worker, launched by tests/test_zzz_adasum_gpu.py::test_adasum_on_real_peers.

With ``B200MPI_ADASUM_KERNEL=1``: ``comm.adasum`` on real peers (up to 64 CTAs per rank), then ``adasum_allreduce_`` through
the kernel; otherwise ``adasum_allreduce_`` through the allgather + torch tree. Every rank generates every rank's inputs and
checks its result bit for bit against tests/adasum_oracle.py. Exits non-zero on any mismatch."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from adasum_oracle import expected, kernel_depth, kernel_geometry, torch_depth  # noqa: E402
from collective_oracle import assert_bits  # noqa: E402
from mpi_operator_b200.hvd.adasum import _kernel_enabled, adasum_allreduce_  # noqa: E402
from mpi_operator_b200.launch.env import rank_info_from_env  # noqa: E402
from mpi_operator_b200.runtime.comm import Communicator  # noqa: E402


def inputs(world, n, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn(n, device="cuda", generator=g)
    return [((0.5 * base + torch.randn(n, device="cuda", generator=g)) * (1.0 + 0.25 * r)).to(dtype) for r in range(world)]


def main():
    info = rank_info_from_env()
    dev = info.local_rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    comm = Communicator.create(info.rank, info.world_size, dev, info.job_id)
    comm.set_tuning(timeout_ms=10000)
    W, R = comm.world, comm.rank
    kernel = _kernel_enabled()
    max_blocks = comm.get_tuning()["max_blocks"]
    fails = 0

    def same(name, got, want):
        nonlocal fails
        try:
            assert_bits(got, want.to(got.device), name)
        except AssertionError as e:
            print(f"[rank {R}] {e}", flush=True)
            fails += 1

    def kernel_want(xs, what):
        _, per, blocks = kernel_geometry(xs[0].numel(), xs[0].dtype, W, max_blocks=max_blocks, emulated=False)
        return expected(xs, xs[0].dtype, depth=kernel_depth(per, blocks, W, xs[0].dtype), what=what)

    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        vn = 4 if dtype == torch.float32 else 8
        for n in (1, 4099, 64 * 512 * vn * W + 3, (1 << 20) + 5):          # the third needs all 64 CTAs per rank
            xs = inputs(W, n, dtype, n)
            what = f"world {W} {dtype} n={n} kernel={int(kernel)}"
            if kernel:
                want = kernel_want(xs, what)
                out = torch.empty_like(xs[R])
                comm.adasum(xs[R].clone(), out)
                torch.cuda.synchronize()
                comm.check_error()
                same(f"comm.adasum {what}", out, want)
            else:
                want = expected(xs, dtype, depth=torch_depth(n), what=what)
            t = xs[R].clone()
            adasum_allreduce_(comm, t)
            torch.cuda.synchronize()
            comm.check_error()
            same(f"adasum_allreduce_ {what}", t, want)
    comm.host_barrier()
    print(f"[rank {R}] adasum_mp_worker done (kernel={int(kernel)}), failures={fails}", flush=True)
    comm.destroy()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
