"""``torch.distributed`` backend ``"b200mpi"``: the second front-end SURVEY.md section 7.1 step 7 names next to the NCCL-ABI
``LD_PRELOAD`` shim ("a c10d ProcessGroup extension ... keep both behind one runtime API").

    import mpi_operator_b200.parallel.c10d_backend        # registers the backend
    torch.distributed.init_process_group("b200mpi")       # RANK / WORLD_SIZE / LOCAL_RANK from torchrun or our mpirun
    model = torch.nn.parallel.DistributedDataParallel(model)

No preloading and no NCCL in the process: the process group is a Python ``ProcessGroup`` whose collectives call the same
runtime the shim calls - ``runtime.comm.Communicator`` (sm_90a NVSwitch kernels, enqueued on the CURRENT CUDA stream, so the
returned ``Work`` is complete in stream order exactly like ProcessGroupNCCL's) for CUDA tensors, the ``libmpi`` shim
(``hvd.host_backend.HostCommunicator``) for CPU tensors. Reference call site that creates the obligation: the workloads of
examples/v2beta1/tensorflow-benchmarks/tensorflow-benchmarks.yaml:26-42 reach their collectives through a framework-level
communication library; with PyTorch that library is c10d.

``new_group(ranks)`` works as well: a sub-group gets communicators of its own on first use - on the host an MPI
sub-communicator made by its members only (``MPI_Comm_create_group``, csrc/mpi_shim/mpi_comm.cc), on the device a separate
runtime communicator whose rendezvous name is derived from the member list.
Reductions: SUM, AVG, MIN, MAX natively, PRODUCT through one allgather. Rooted operations (``gather``, ``scatter``, ``reduce``) ride
the unrooted kernels; ``send`` / ``recv`` / ``batch_isend_irecv`` and the uneven list form of ``all_to_all`` use the libmpi shim's
tagged mailboxes (CUDA tensors: the runtime's point-to-point kernel when the communicator has it, staged through the host otherwise).
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch
import torch.distributed as dist
from torch._C._distributed_c10d import (AllgatherOptions, AllreduceOptions, AllToAllOptions, BarrierOptions, BroadcastOptions, GatherOptions,
                                        ReduceOp, ReduceOptions, ReduceScatterOptions, ScatterOptions, _create_work_from_future)
from torch.futures import Future

BACKEND_NAME = "b200mpi"
_OP_NAMES = ((ReduceOp.SUM, "sum"), (ReduceOp.AVG, "avg"), (ReduceOp.MIN, "min"), (ReduceOp.MAX, "max"))


def _op_name(op) -> Optional[str]:
    """AllreduceOptions.reduceOp is a ReduceOp OBJECT (it can carry a premul-sum factor): compare, do not hash."""
    for cand, name in _OP_NAMES:
        if op == cand:
            return name
    return None


def _done(result):
    fut: Future = Future()
    fut.set_result(result)
    return _create_work_from_future(fut)


def _bcast_opts(root: int):
    o = BroadcastOptions()
    o.rootRank = root
    return o


_world_host = None   # the process-wide MPI_COMM_WORLD communicator of the libmpi shim (MPI_Init happens once per process)


def _host_world(rank: int, world: int):
    global _world_host
    if _world_host is None:
        from ..hvd.host_backend import HostCommunicator
        from ..launch.env import job_id_from_env
        os.environ.setdefault("B200MPI_JOB_ID", job_id_from_env(os.environ))
        os.environ.setdefault("B200MPI_RANK", str(rank))
        os.environ.setdefault("B200MPI_WORLD_SIZE", str(world))
        _world_host = HostCommunicator()
        import atexit
        atexit.register(_finalize_host)   # MPI_Finalize: rank 0 unlinks the job's rendezvous segment (no launcher of ours may be around to do it)
        if (_world_host.rank, _world_host.world) != (rank, world):
            raise RuntimeError(f"b200mpi backend: the MPI shim sees rank {_world_host.rank}/{_world_host.world}, "
                               f"torch.distributed {rank}/{world}")
    return _world_host


_dev_comms: list = []


def _finalize_dev() -> None:
    while _dev_comms:
        c = _dev_comms.pop()
        try:
            c.destroy()
        except Exception:  # noqa: BLE001
            pass


def _finalize_host() -> None:
    global _world_host
    c, _world_host = _world_host, None
    if c is not None:
        try:
            c.destroy()
        except Exception:  # noqa: BLE001
            pass


class B200ProcessGroup(dist.ProcessGroup):
    def __init__(self, rank: int, world_size: int, global_ranks: Optional[List[int]] = None, global_rank: Optional[int] = None,
                 global_world: Optional[int] = None):
        super().__init__(rank, world_size)
        self._rank, self._world = rank, world_size
        self._granks = list(global_ranks) if global_ranks else None          # None: the group is the whole world, in order
        self._grank = rank if global_rank is None else global_rank
        self._gworld = world_size if global_world is None else global_world
        if self._granks == list(range(self._gworld)):
            self._granks = None
        self._host = None     # hvd.host_backend.HostCommunicator (CPU tensors), created on first use
        self._dev = None      # runtime.comm.Communicator (CUDA tensors), created on first use

    # ------------------------------------------------------------ plumbing --
    def size(self):
        return self._world

    def rank(self):
        return self._rank

    def getBackendName(self):  # noqa: N802
        return BACKEND_NAME

    def __repr__(self):
        return f"B200ProcessGroup(rank={self._rank}, world={self._world})"

    def _comm(self, t: torch.Tensor):
        from ..launch.env import job_id_from_env
        import zlib
        digest = 0 if self._granks is None else zlib.crc32(",".join(map(str, self._granks)).encode())
        if t.is_cuda:
            if self._dev is None:
                from ..runtime.comm import Communicator
                dev = t.device.index if t.device.index is not None else torch.cuda.current_device()
                name = job_id_from_env(os.environ) + ("-c10d" if self._granks is None else f"-c10d-{digest:08x}")
                self._dev = Communicator.create(self._rank, self._world, dev, name)
                _dev_comms.append(self._dev)
                if len(_dev_comms) == 1:
                    import atexit
                    atexit.register(_finalize_dev)    # rank 0 unlinks the rendezvous segments
            return self._dev
        if self._host is None:
            world = _host_world(self._grank, self._gworld)
            self._host = world if self._granks is None else world.sub(self._granks, tag=digest)
            if self._host is None or (self._host.rank, self._host.world) != (self._rank, self._world):
                raise RuntimeError("b200mpi backend: sub-communicator does not match the torch.distributed group")
        return self._host

    @staticmethod
    def _contig(t: torch.Tensor):
        return t if t.is_contiguous() else t.contiguous()

    def _allreduce_one(self, t: torch.Tensor, op) -> None:
        c = self._comm(t)
        if self._world == 1:
            return
        if op == ReduceOp.PRODUCT:
            w = self._contig(t)
            g = torch.empty((self._world,) + tuple(w.shape), dtype=w.dtype, device=w.device)
            c.allgather(w, g)
            t.copy_(g.prod(0))
            return
        name = _op_name(op)
        if name is None:
            raise NotImplementedError(f"b200mpi backend: reduction {op} is not supported (SUM, AVG, MIN, MAX, PRODUCT)")
        w = self._contig(t)
        if w.is_cuda and w.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            f = w.float()                                   # the device kernels reduce floating point; integers round-trip (exact below 2^24)
            c.allreduce(f, f, op=name)
            t.copy_(f.to(t.dtype))
            return
        c.allreduce(w, w, op=name)
        if w is not t:
            t.copy_(w)

    # --------------------------------------------------------- collectives --
    def allreduce(self, tensors: List[torch.Tensor], opts=AllreduceOptions()):
        with torch.no_grad():
            for t in tensors:
                self._allreduce_one(t.detach(), opts.reduceOp)
        return _done(tensors)

    def allreduce_coalesced(self, tensors: List[torch.Tensor], opts=AllreduceOptions()):
        return self.allreduce(tensors, opts)

    def reduce(self, tensors: List[torch.Tensor], opts=ReduceOptions()):
        # every rank ends up with the result; only the root's copy is defined by the API
        with torch.no_grad():
            for t in tensors:
                self._allreduce_one(t.detach(), opts.reduceOp)
        return _done(tensors)

    def broadcast(self, tensors: List[torch.Tensor], opts=BroadcastOptions()):
        with torch.no_grad():
            for t in tensors:
                c = self._comm(t)
                if self._world == 1:
                    continue
                w = self._contig(t.detach())
                c.broadcast(w, root=opts.rootRank)
                if w.data_ptr() != t.data_ptr():
                    t.detach().copy_(w)
        return _done(tensors)

    def _allgather_base(self, output: torch.Tensor, inp: torch.Tensor, opts=AllgatherOptions()):
        with torch.no_grad():
            c = self._comm(inp)
            src = self._contig(inp.detach())
            if self._world == 1:
                output.detach().view(-1).copy_(src.view(-1))
            else:
                out = output.detach()
                dst = out if out.is_contiguous() else torch.empty_like(out, memory_format=torch.contiguous_format)
                flat_in = src.view(-1)
                pad = flat_in.numel() * flat_in.element_size() % 2   # the device allgather moves 2-byte units
                if pad and src.is_cuda:
                    raise NotImplementedError("b200mpi backend: allgather of an odd number of bytes on CUDA tensors")
                c.allgather(flat_in, dst.view(-1))
                if dst is not out:
                    out.copy_(dst)
        return _done(output)

    def allgather(self, output_lists: List[List[torch.Tensor]], inputs: List[torch.Tensor], opts=AllgatherOptions()):
        with torch.no_grad():
            for outs, inp in zip(output_lists, inputs):
                src = self._contig(inp.detach())
                flat = torch.empty(self._world * src.numel(), dtype=src.dtype, device=src.device)
                self._allgather_base(flat, src, opts)
                for r, o in enumerate(outs):
                    o.detach().copy_(flat[r * src.numel():(r + 1) * src.numel()].view_as(src))
        return _done(output_lists)

    def allgather_into_tensor_coalesced(self, outputs, inputs, opts=AllgatherOptions()):
        for o, i in zip(outputs, inputs):
            self._allgather_base(o, i, opts)
        return _done(outputs)

    def _reduce_scatter_base(self, output: torch.Tensor, inp: torch.Tensor, opts=ReduceScatterOptions()):
        with torch.no_grad():
            c = self._comm(inp)
            src = self._contig(inp.detach())
            if self._world == 1:
                output.detach().view(-1).copy_(src.view(-1))
                return _done(output)
            op = opts.reduceOp
            name = _op_name(op)
            if name is None or (src.is_cuda and src.dtype not in (torch.float32, torch.bfloat16, torch.float16)):
                full = src.clone()                          # generic: allreduce, keep the own block
                self._allreduce_one(full, op)
                output.detach().copy_(full.view(self._world, -1)[self._rank].view_as(output))
                return _done(output)
            out = output.detach()
            dst = out if out.is_contiguous() else torch.empty_like(out, memory_format=torch.contiguous_format)
            c.reduce_scatter(src.view(-1), dst.view(-1), op=name)
            if dst is not out:
                out.copy_(dst)
        return _done(output)

    def reduce_scatter(self, outputs: List[torch.Tensor], input_lists: List[List[torch.Tensor]], opts=ReduceScatterOptions()):
        for out, ins in zip(outputs, input_lists):
            self._reduce_scatter_base(out, torch.cat([self._contig(t.detach()).view(-1) for t in ins]), opts)
        return _done(outputs)

    def reduce_scatter_tensor_coalesced(self, outputs, inputs, opts=ReduceScatterOptions()):
        for o, i in zip(outputs, inputs):
            self._reduce_scatter_base(o, i, opts)
        return _done(outputs)

    def alltoall_base(self, output: torch.Tensor, inp: torch.Tensor, output_split_sizes: Optional[List[int]],
                      input_split_sizes: Optional[List[int]], opts=AllToAllOptions()):
        if output_split_sizes or input_split_sizes:
            raise NotImplementedError("b200mpi backend: all_to_all_single with uneven splits (use hvd.alltoall(tensor, splits))")
        with torch.no_grad():
            c = self._comm(inp)
            src = self._contig(inp.detach())
            if self._world == 1:
                output.detach().copy_(src.view_as(output))
            else:
                out = output.detach()
                dst = out if out.is_contiguous() else torch.empty_like(out, memory_format=torch.contiguous_format)
                c.alltoall(src, dst)
                if dst is not out:
                    out.copy_(dst)
        return _done(output)

    def alltoall(self, output_tensors: List[torch.Tensor], input_tensors: List[torch.Tensor], opts=AllToAllOptions()):
        """List form (``dist.all_to_all``): one tensor per peer. Equal sizes ride the all-to-all kernel; uneven lists exchange
        pairwise (rank r sends to r+k and receives from r-k in round k: every pair meets once, nobody waits in a cycle)."""
        with torch.no_grad():
            n = {t.numel() * t.element_size() for t in list(input_tensors) + list(output_tensors)}
            if len(n) == 1 and len({t.dtype for t in input_tensors}) == 1:
                src = torch.cat([self._contig(t.detach()).view(-1) for t in input_tensors])
                dst = torch.empty_like(src)
                self.alltoall_base(dst, src, None, None, opts)
                per = src.numel() // self._world
                for r, o in enumerate(output_tensors):
                    o.detach().copy_(dst[r * per:(r + 1) * per].view_as(o))
            else:
                output_tensors[self._rank].detach().copy_(input_tensors[self._rank].detach())
                for k in range(1, self._world):
                    to, frm = (self._rank + k) % self._world, (self._rank - k) % self._world
                    self._p2p(input_tensors[to], to, 0, True)       # eager send: buffered at the receiver, returns at once
                    self._p2p(output_tensors[frm], frm, 0, False)
        return _done(output_tensors)

    def gather(self, output_lists: List[List[torch.Tensor]], input_tensors: List[torch.Tensor], opts=GatherOptions()):
        # one allgather; only the root copies the blocks out (every rank passes a tensor of the same shape, the API's contract)
        with torch.no_grad():
            for k, inp in enumerate(input_tensors):
                src = self._contig(inp.detach())
                flat = torch.empty(self._world * src.numel(), dtype=src.dtype, device=src.device)
                self._allgather_base(flat, src)
                if self._rank == opts.rootRank:
                    for r, o in enumerate(output_lists[k]):
                        o.detach().copy_(flat[r * src.numel():(r + 1) * src.numel()].view_as(o))
        return _done(output_lists)

    def scatter(self, output_tensors: List[torch.Tensor], input_lists: List[List[torch.Tensor]], opts=ScatterOptions()):
        # the root's list travels as one broadcast; every rank keeps its own block
        with torch.no_grad():
            for k, out in enumerate(output_tensors):
                o = out.detach()
                flat = torch.empty(self._world * o.numel(), dtype=o.dtype, device=o.device)
                if self._rank == opts.rootRank:
                    flat.copy_(torch.cat([self._contig(t.detach()).view(-1) for t in input_lists[k]]))
                self.broadcast([flat], _bcast_opts(opts.rootRank))
                o.copy_(flat[self._rank * o.numel():(self._rank + 1) * o.numel()].view_as(o))
        return _done(output_tensors)

    def _p2p(self, t: torch.Tensor, peer: int, tag: int, is_send: bool) -> None:
        """CUDA tensors use the runtime's point-to-point kernel when the communicator was created with it (B200MPI_P2P=1);
        otherwise - and for CPU tensors - the bytes travel through the libmpi shim's mailboxes (tag matching, eager sends)."""
        td = t.detach()
        if td.is_cuda:
            c = self._comm(td)
            if getattr(c, "has_p2p", False) and td.is_contiguous():
                (c.send if is_send else c.recv)(td, peer)
                return
            host = self._comm(torch.empty(0))
            if is_send:
                host.send(td.contiguous().cpu(), peer, tag)
            else:
                tmp = torch.empty(td.shape, dtype=td.dtype, device="cpu")
                host.recv(tmp, peer, tag)
                td.copy_(tmp)
            return
        host = self._comm(td)
        if is_send:
            host.send(self._contig(td), peer, tag)
        elif td.is_contiguous():
            host.recv(td, peer, tag)
        else:
            tmp = torch.empty(td.shape, dtype=td.dtype)
            host.recv(tmp, peer, tag)
            td.copy_(tmp)

    def send(self, tensors: List[torch.Tensor], dst_rank: int, tag: int = 0):
        with torch.no_grad():
            for t in tensors:
                self._p2p(t, dst_rank, tag, True)
        return _done(None)

    def recv(self, tensors: List[torch.Tensor], src_rank: int, tag: int = 0):
        with torch.no_grad():
            for t in tensors:
                self._p2p(t, src_rank, tag, False)
        return _done(None)

    def barrier(self, opts=BarrierOptions()):
        if self._world > 1:
            c = self._dev if self._dev is not None else self._comm(torch.empty(0))
            if c is self._dev:
                torch.cuda.synchronize()
                c.host_barrier()
            else:
                c.barrier()
        return _done(None)

    def shutdown(self):
        if self._dev in _dev_comms:
            _dev_comms.remove(self._dev)
        for c in (self._dev, self._host if self._host is not _world_host else None):   # MPI itself ends with the process
            if c is not None:
                try:
                    c.destroy()
                except Exception:  # noqa: BLE001
                    pass
        self._dev = self._host = None


def _create(dist_opts, backend_opts):
    ranks = list(getattr(dist_opts, "global_ranks_in_group", []) or [])
    gworld = dist.get_world_size() if dist.is_initialized() else dist_opts.group_size
    grank = ranks[dist_opts.group_rank] if ranks else dist_opts.group_rank
    return B200ProcessGroup(dist_opts.group_rank, dist_opts.group_size, ranks or None, grank, gworld)


def register() -> None:
    if BACKEND_NAME.upper() not in getattr(dist.Backend, "backend_list", []) and BACKEND_NAME not in getattr(dist.Backend, "backend_list", []):
        dist.Backend.register_backend(BACKEND_NAME, _create, extended_api=True, devices=["cpu", "cuda"])


register()
