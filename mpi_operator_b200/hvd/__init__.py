"""Horovod-compatible front-end over the b200mpi runtime.

The reference's workloads call Horovod (examples/v2beta1/horovod/
tensorflow_mnist.py:90 ``hvd.init()``, :123-130 LR x ``hvd.size()``, :133
``hvd.DistributedOptimizer(opt, op=hvd.Average)``, :143 broadcast from rank 0,
:155 GPU pinning by ``hvd.local_rank()``, :159 rank-0-only checkpoints; and
``--variable_update=horovod`` in tensorflow-benchmarks.yaml:42).  Horovod's C++
core is replaced twice over.  For the training hot path: gradients living in a
symmetric window (no fusion-buffer copies), bucket allreduce kernels with the
average fused in, launched from autograd hooks on a high-priority stream
(``DistributedOptimizer``).  For everything else Horovod's background thread
does — named tensors submitted in any order, ``*_async`` handles, fusion of many
small tensors, response cache, timeline, stall inspector, ``join()`` — the native
``hvdcore`` engine (csrc/hvd_core, ``hvd/engine.py``).  Usage is the
``horovod.torch`` one:

    import mpi_operator_b200.hvd as hvd      # or: import horovod.torch as hvd
    hvd.init(); torch.cuda.set_device(hvd.local_rank())
    opt = hvd.DistributedOptimizer(opt, named_parameters=model.named_parameters())
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
"""
from __future__ import annotations

import os


from ..launch.env import rank_info_from_env
from .exceptions import HorovodInternalError, HostsUpdatedInterrupt  # noqa: F401

Average, Sum, Adasum, Min, Max, Product = "average", "sum", "adasum", "min", "max", "product"

_state = {"comm": None, "info": None, "engine": None, "optimizers": []}


class HorovodNotInitialized(RuntimeError):
    pass


def _comm():
    if _state["comm"] is None:
        raise HorovodNotInitialized("hvd.init() has not been called")
    return _state["comm"]


def _elastic_generation() -> int:
    return int(os.environ.get("B200MPI_GENERATION", "0") or 0)


def _job_id(info) -> str:
    """Rendezvous key of the CURRENT incarnation of the world: the launcher's job id, plus the elastic generation when the
    world is being re-formed in place (survivors and newly spawned ranks meet under the new key)."""
    g = _elastic_generation()
    return info.job_id + (f"-g{g}" if g else "")


def _announce_ready() -> None:
    """Ranks spawned into a running elastic job tell the launcher they are about to join (imports done): only then does it
    publish the new world to the survivors, which keep training on the old one in the meantime."""
    d, g = os.environ.get("B200MPI_ELASTIC_DIR"), _elastic_generation()
    if d and g and os.environ.get("B200MPI_ELASTIC_JOIN") == "1":
        try:
            with open(os.path.join(d, f"ready.{g}.{os.environ.get('B200MPI_RANK', '0')}"), "w") as f:
                f.write("ready\n")
        except OSError:
            pass


def init(comm=None) -> None:
    """Join the job's rendezvous; device = LOCAL_RANK (set it first with torch.cuda.set_device if you prefer)."""
    if _state["comm"] is not None:
        return
    import torch
    from ..runtime.comm import Communicator
    info = rank_info_from_env()
    _state["info"] = info
    if comm is not None:
        _state["comm"] = comm
        return
    _announce_ready()
    if _elastic_generation() and not os.environ.get("B200MPI_TIMEOUT_MS"):
        os.environ.setdefault("B200MPI_INIT_TIMEOUT_MS", "180000")   # survivors join at their next commit, not immediately
    if not torch.cuda.is_available() or os.environ.get("B200MPI_HVD_DEVICE", "") == "cpu":
        # CPU job (the reference's Horovod MNIST example runs on CPU workers): collectives over the libmpi shim
        from .host_backend import HostCommunicator
        if _elastic_generation():
            os.environ["B200MPI_JOB_ID"] = _job_id(info)     # the libmpi shim reads the key from the environment
            os.environ.setdefault("B200MPI_TIMEOUT_MS", "180000")
        try:
            _state["comm"] = HostCommunicator()
        finally:
            os.environ["B200MPI_JOB_ID"] = info.job_id
        _start_engine(info, None)
        return
    dev = info.local_rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    _state["comm"] = Communicator.create(info.rank, info.world_size, dev, _job_id(info))
    _start_engine(info, dev)


def _reinit(world: int, generation: int) -> None:
    """Elastic rescale IN PLACE: this (surviving) rank leaves the old world and joins generation `generation` with `world`
    ranks, keeping its process, its CUDA context and its model. Optimizers built by ``DistributedOptimizer`` re-home their
    gradient windows into the new communicator."""
    opts = [o for o in (r() for r in _state.get("optimizers", [])) if o is not None]
    for o in opts:
        o._detach()
    base_job = _state["info"].job_id if _state.get("info") else rank_info_from_env().job_id
    base_job = os.environ.get("B200MPI_BASE_JOB_ID", base_job)
    os.environ.setdefault("B200MPI_BASE_JOB_ID", base_job)
    e = _state["engine"]
    if e is not None:
        _state["engine"] = None
        e.shutdown()
    c = _state["comm"]
    for k in ("B200MPI_WORLD_SIZE", "OMPI_COMM_WORLD_SIZE", "PMI_SIZE", "WORLD_SIZE", "HOROVOD_SIZE", "B200MPI_LOCAL_SIZE",
              "OMPI_COMM_WORLD_LOCAL_SIZE", "MPI_LOCALNRANKS", "LOCAL_WORLD_SIZE", "HOROVOD_LOCAL_SIZE"):
        if k in os.environ:
            os.environ[k] = str(world)
    os.environ["B200MPI_GENERATION"] = str(generation)
    os.environ["B200MPI_JOB_ID"] = base_job
    os.environ.pop("B200MPI_ELASTIC_JOIN", None)
    if not os.environ.get("B200MPI_TIMEOUT_MS_USER"):
        os.environ.setdefault("B200MPI_INIT_TIMEOUT_MS", "180000")
    info = rank_info_from_env()
    _state["info"] = info
    if hasattr(c, "reinit"):          # host backend: the libmpi shim re-attaches under the new key
        os.environ["B200MPI_JOB_ID"] = _job_id(info)
        os.environ.setdefault("B200MPI_TIMEOUT_MS", "180000")
        c.reinit()
        os.environ["B200MPI_JOB_ID"] = base_job
        _start_engine(info, None)
    else:
        import torch
        from ..runtime.comm import Communicator
        torch.cuda.synchronize()
        dev = c.device
        c.destroy()
        _state["comm"] = Communicator.create(info.rank, info.world_size, dev, _job_id(info))
        _start_engine(info, dev)
    for o in opts:
        o._attach()


_atexit_registered = False


def _start_engine(info, dev) -> None:
    """Native background engine (hvd/engine.py). Host tensors: on unless B200MPI_HVD_ENGINE=0. Device tensors: only with
    B200MPI_HVD_ENGINE=1 (multi-GPU only, not yet run on H100; the direct path stays the default); it gets a communicator of its own because
    collectives on one communicator must be issued in the same order on every rank."""
    global _atexit_registered
    want = os.environ.get("B200MPI_HVD_ENGINE", "")
    if want == "0" or (dev is not None and want != "1"):
        return
    from .engine import Engine
    gcomm = None
    if dev is not None:
        from ..runtime.comm import Communicator
        gcomm = Communicator.create(info.rank, info.world_size, dev, _job_id(info) + "-hvdgpu")
    _state["engine"] = Engine(_job_id(info), info.rank, info.world_size, gcomm)
    if not _atexit_registered:   # a script that forgets hvd.shutdown() must not leave its peers negotiating with a ghost
        import atexit
        atexit.register(shutdown)
        _atexit_registered = True


def _dump_engine_stats(e) -> None:
    """Per-rank engine counters for the operator's /metrics (the node agent harvests $B200MPI_STATS_DIR when the pod ends)."""
    d = os.environ.get("B200MPI_STATS_DIR")
    if not d:
        return
    try:
        import json
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, f"stats-hvd-rank{e.rank}-{os.getpid()}.json")
        with open(path + ".tmp", "w") as f:
            json.dump({"rank": e.rank, "world": e.world, "ops": [], "hvd": e.stats()}, f)
        os.replace(path + ".tmp", path)
    except OSError:
        pass


def shutdown() -> None:
    e = _state["engine"]
    if e is not None:
        _state["engine"] = None
        _dump_engine_stats(e)
        e.shutdown()
    for pid, ps in list(_process_sets.items()):
        if pid:
            remove_process_set(ps)
    _next_process_set_id[0] = 1
    c = _state["comm"]
    if c is not None:
        c.destroy()
    _state["comm"] = None


def is_initialized() -> bool:
    return _state["comm"] is not None


def rank() -> int: return _comm().rank  # noqa: E704
def size() -> int: return _comm().world  # noqa: E704
def local_rank() -> int: return _state["info"].local_rank  # noqa: E704
def local_size() -> int: return _state["info"].local_size  # noqa: E704
def cross_rank() -> int: return 0  # noqa: E704  (single box)
def cross_size() -> int: return 1  # noqa: E704
def mpi_threads_supported() -> bool: return False  # noqa: E704
def mpi_built() -> bool: return True  # noqa: E704
def mpi_enabled() -> bool: return True  # noqa: E704
def gloo_built() -> bool: return False  # noqa: E704
def gloo_enabled() -> bool: return False  # noqa: E704
def nccl_built() -> int: return 1  # noqa: E704  (tensorflow_mnist.py:127 checks this before Adasum)
def cuda_built() -> bool:
    import torch
    return torch.cuda.is_available()
def rocm_built() -> bool: return False  # noqa: E704
def ddl_built() -> bool: return False  # noqa: E704
def ccl_built() -> bool: return False  # noqa: E704


def _op_name(op, average):
    if average is not None:
        return "avg" if average else "sum"
    if op in (None, Average):
        return "avg"
    if op == Sum:
        return "sum"
    if op == Min:
        return "min"
    if op == Max:
        return "max"
    if op == Adasum:
        return "adasum"
    if op == Product:
        return "prod"
    raise ValueError(f"unknown reduction op {op!r}")


class ProcessSet:
    """Horovod >= 0.23 process sets (beyond the reference's Horovod 0.19 / 0.20, kept because newer Horovod scripts use them):
    a subset of the job's ranks with a communicator of its own. ``hvd.global_process_set`` is every rank; others are made
    with ``hvd.add_process_set([ranks])`` - on the host an MPI sub-communicator formed by its members
    (``MPI_Comm_create_group``, csrc/mpi_shim/mpi_comm.cc), on GPUs a separate runtime communicator. Collectives that take
    ``process_set=`` run on that communicator through the direct (call-order) path; ``root_rank`` stays a GLOBAL rank."""

    def __init__(self, ranks=None):
        self._ranks = None if ranks is None else sorted(int(r) for r in set(ranks))
        self.process_set_id = 0 if ranks is None else None
        self._c = None

    @property
    def ranks(self):
        return list(range(_comm_world().world)) if self._ranks is None else list(self._ranks)

    def size(self) -> int:
        return len(self.ranks)

    def included(self) -> bool:
        return self._ranks is None or _comm_world().rank in self._ranks

    def rank(self) -> int:
        """This process's rank inside the set (-1 when it is not a member)."""
        me = _comm_world().rank
        return me if self._ranks is None else (self._ranks.index(me) if me in self._ranks else -1)

    def __repr__(self):
        return f"ProcessSet(id={self.process_set_id}, ranks={self.ranks if _state['comm'] is not None else self._ranks})"


global_process_set = ProcessSet()
_process_sets = {0: global_process_set}
_next_process_set_id = [1]


def _comm_world():
    return _state.get("world_comm") or _comm()


def add_process_set(process_set) -> ProcessSet:
    """Register a process set (a ``ProcessSet`` or a list of ranks). Every rank of the job calls this, in the same order (the ids
    must agree); the members build the set's communicator."""
    ps = process_set if isinstance(process_set, ProcessSet) else ProcessSet(process_set)
    if ps._ranks is None:
        return global_process_set
    world = _comm_world()
    if not ps._ranks or ps._ranks[0] < 0 or ps._ranks[-1] >= world.world:
        raise ValueError(f"process set ranks {ps._ranks} are outside the job's 0..{world.world - 1}")
    for other in _process_sets.values():
        if other._ranks == ps._ranks:
            raise ValueError(f"a process set with ranks {ps._ranks} already exists (id {other.process_set_id})")
    ps.process_set_id = _next_process_set_id[0]
    _next_process_set_id[0] += 1
    if ps.included():
        if getattr(world, "device", None) == "cpu":
            ps._c = world.sub(ps._ranks, tag=1000 + ps.process_set_id)
        else:
            from ..runtime.comm import Communicator
            ps._c = Communicator.create(ps._ranks.index(world.rank), len(ps._ranks), world.device,
                                        f"{_state['info'].job_id}-ps{ps.process_set_id}")
    _process_sets[ps.process_set_id] = ps
    return ps


def remove_process_set(process_set) -> bool:
    if process_set is global_process_set:
        raise ValueError("the global process set cannot be removed")
    pid = getattr(process_set, "process_set_id", None)
    if pid is None or _process_sets.get(pid) is not process_set:
        return False
    del _process_sets[pid]
    if process_set._c is not None:
        try:
            process_set._c.destroy()
        except Exception:  # noqa: BLE001
            pass
        process_set._c = None
    process_set.process_set_id = None
    return True


class _in_process_set:
    """``with _in_process_set(ps):`` - the collectives below run on the set's communicator: the module-level communicator is
    swapped for the duration of the call (and the engine switched off: process-set collectives take the call-order path), so
    ``size()`` / ``rank()`` inside the implementation mean the set's. Not re-entrant across threads, like Horovod's Python API."""

    def __init__(self, ps):
        self.ps = None if (ps is None or ps is global_process_set) else ps

    def __enter__(self):
        ps = self.ps
        if ps is None:
            return self
        if ps.process_set_id is None or _process_sets.get(ps.process_set_id) is not ps:
            raise ValueError("this process set is not registered: call hvd.add_process_set(process_set) on every rank first")
        if not ps.included():
            raise ValueError(f"rank {_comm_world().rank} is not part of process set {ps.process_set_id} (ranks {ps.ranks})")
        self.saved = (_state["comm"], _state["engine"], _state.get("world_comm"))
        _state["world_comm"] = self.saved[2] or self.saved[0]
        _state["comm"], _state["engine"] = ps._c, None
        return self

    def __exit__(self, *exc):
        if self.ps is not None:
            _state["comm"], _state["engine"], _state["world_comm"] = self.saved
        return False

    def root(self, root_rank: int) -> int:
        """Horovod's root_rank is a global rank; the communicator wants the rank inside the set."""
        if self.ps is None:
            return root_rank
        if root_rank not in self.ps._ranks:
            raise ValueError(f"root_rank {root_rank} is not part of process set {self.ps.process_set_id} (ranks {self.ps.ranks})")
        return self.ps._ranks.index(root_rank)


def _check_process_set(ps) -> None:   # kept for callers that only accept the global set
    if ps is not None and ps is not global_process_set:
        raise NotImplementedError("this operation only supports hvd.global_process_set")


class _Done:
    """Handle of an operation that already completed in stream order (direct path)."""

    def __init__(self, result):
        self.result = result

    def done(self) -> bool:
        return True

    def wait(self):
        return self.result


def _engine_for(tensor):
    e = _state["engine"]
    if e is None or (tensor.is_cuda and not e.has_gpu):
        return None
    return e


def allreduce(tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    out = tensor.clone()
    allreduce_(out, average, name, op, prescale_factor, postscale_factor, process_set)
    return out


def allreduce_(tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    return allreduce_async_(tensor, average, name, op, prescale_factor, postscale_factor, process_set).wait()


def allreduce_async(tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    return allreduce_async_(tensor.clone(), average, name, op, prescale_factor, postscale_factor, process_set)


def allreduce_async_(tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    if process_set is not None and process_set is not global_process_set:
        with _in_process_set(process_set):
            return allreduce_async_(tensor, average, name, op, prescale_factor, postscale_factor)
    return _allreduce_async_impl(tensor, average, name, op, prescale_factor, postscale_factor)


def _allreduce_async_impl(tensor, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0):
    """In-place allreduce; returns a handle for ``synchronize`` / ``poll``. With the engine, ranks may submit named
    tensors in different orders and small tensors submitted close together travel fused."""
    import torch
    opn = _op_name(op, average)
    if opn == "adasum":
        e = _engine_for(tensor)
        if e is not None and not tensor.is_cuda and tensor.is_floating_point() and tensor.dtype in (torch.float32, torch.float64, torch.float16, torch.bfloat16):
            # native: every rank's vector in a shared scratch segment, all ranks work on their 1/W slice of every pair of a
            # tree level (csrc/hvd_core/hvd_core.cc: host_adasum); negotiated by name like any other engine collective
            t = tensor if tensor.is_contiguous() else tensor.contiguous()
            h = e.allreduce_async(t, t, name, "adasum", prescale_factor, postscale_factor)
            h.result = tensor
            if t is not tensor:
                h.post = lambda _r, _t=t, _o=tensor: _o.copy_(_t)
            return h
        from .adasum import adasum_allreduce_   # device tensors: one allgather kernel + a local fp32 tree
        if prescale_factor != 1.0:
            tensor.mul_(prescale_factor)
        adasum_allreduce_(_comm(), tensor)
        if postscale_factor != 1.0:
            tensor.mul_(postscale_factor)
        return _Done(tensor)
    if opn == "prod" and tensor.is_cuda:
        # the device kernels reduce with sum / min / max; a product is one allgather kernel + a local reduction
        t = tensor.contiguous()
        g = torch.empty((size(),) + tuple(t.shape), dtype=t.dtype, device=t.device)
        _comm().allgather(t if prescale_factor == 1.0 else t * prescale_factor, g)
        tensor.copy_(g.prod(0) if postscale_factor == 1.0 else g.prod(0) * postscale_factor)
        return _Done(tensor)
    e = _engine_for(tensor)
    if e is not None:
        t = tensor if tensor.is_contiguous() else tensor.contiguous()
        if tensor.is_cuda and (t.dtype not in (torch.float32, torch.bfloat16, torch.float16) or opn == "prod"):
            t = t.float()        # the device kernels reduce floating point; integers round-trip through fp32
        h = e.allreduce_async(t, t, name, opn, prescale_factor, postscale_factor)
        h.result = tensor
        if t is not tensor:
            h.post = lambda _r, _t=t, _o=tensor: _o.copy_(_t.to(_o.dtype))
        return h
    t = tensor if tensor.is_contiguous() else tensor.contiguous()
    if _on_gpu() and t.dtype not in (torch.float32, torch.bfloat16, torch.float16):   # the host backend reduces every MPI type natively
        f = t.float()
        _comm().allreduce(f, f, op=opn, scale=prescale_factor * postscale_factor)
        tensor.copy_(f.to(tensor.dtype))
        return _Done(tensor)
    _comm().allreduce(t, t, op=opn, scale=prescale_factor * postscale_factor)
    if t is not tensor:
        tensor.copy_(t)
    return _Done(tensor)


def grouped_allreduce(tensors, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    hs = grouped_allreduce_async(tensors, average, name, op, prescale_factor, postscale_factor, process_set)
    return [h.wait() for h in hs]


def grouped_allreduce_async(tensors, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    """All tensors are submitted before any is waited for, so the engine negotiates them in one cycle and fuses them."""
    return [allreduce_async(t, average, f"{name}.{i}" if name else None, op, prescale_factor, postscale_factor, process_set)
            for i, t in enumerate(tensors)]


def grouped_allreduce_(tensors, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    hs = grouped_allreduce_async_(tensors, average, name, op, prescale_factor, postscale_factor, process_set)
    return [h.wait() for h in hs]


def grouped_allreduce_async_(tensors, average=None, name=None, op=None, prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    """In-place form of ``grouped_allreduce_async``."""
    return [allreduce_async_(t, average, f"{name}.{i}" if name else None, op, prescale_factor, postscale_factor, process_set)
            for i, t in enumerate(tensors)]


def grouped_allgather(tensors, name=None, process_set=None):
    with _in_process_set(process_set):
        return [h.wait() for h in grouped_allgather_async(tensors, name)]


def grouped_allgather_async(tensors, name=None):
    return [allgather_async(t, f"{name}.{i}" if name else None) for i, t in enumerate(tensors)]


def allgather(tensor, name=None, process_set=None):
    with _in_process_set(process_set):
        return allgather_async(tensor, name).wait()


def allgather_async(tensor, name=None):
    """Concatenation along the first dimension. Through the engine (host tensors) the first dimensions may differ."""
    import torch
    e = _engine_for(tensor)
    if e is not None and not tensor.is_cuda:
        return e.allgather_async(tensor if tensor.dim() else tensor.reshape(1), name)
    t = tensor.contiguous() if tensor.dim() else tensor.reshape(1)
    n = size()
    # direct path: the ranks first tell each other their first dimension (one 8-byte allgather), equal sizes then take the
    # single-kernel path, ragged ones are padded to the largest and trimmed after the gather (Horovod semantics: concatenation
    # along dim 0 with per-rank first dimensions)
    mine = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    rows = torch.empty(n, dtype=torch.int64, device=t.device)
    _comm().allgather(mine, rows)
    rows = rows.tolist()
    if len(set(rows)) == 1:
        out = torch.empty((n * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        if out.numel():
            _comm().allgather(t, out)
        return _Done(out)
    width = max(rows)
    padded = torch.zeros((width,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    padded[:t.shape[0]] = t
    got = torch.empty((n * width,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    _comm().allgather(padded, got)
    got = got.view((n, width) + tuple(t.shape[1:]))
    return _Done(torch.cat([got[k, :rows[k]] for k in range(n)], dim=0))


def broadcast(tensor, root_rank, name=None, process_set=None):
    out = tensor.clone()
    return broadcast_(out, root_rank, name, process_set)


def broadcast_(tensor, root_rank, name=None, process_set=None):
    with _in_process_set(process_set) as ctx:
        return broadcast_async_(tensor, ctx.root(root_rank), name).wait()


def broadcast_async(tensor, root_rank, name=None):
    return broadcast_async_(tensor.clone(), root_rank, name)


def broadcast_async_(tensor, root_rank, name=None):
    t = tensor if tensor.is_contiguous() else tensor.contiguous()
    e = _engine_for(tensor)
    if e is not None:
        h = e.broadcast_async(t, root_rank, name)
        h.result = tensor
        if t is not tensor:
            h.post = lambda _r, _t=t, _o=tensor: _o.copy_(_t)
        return h
    _comm().broadcast(t, root=root_rank)
    if t is not tensor:
        tensor.copy_(t)
    return _Done(tensor)


def alltoall(tensor, splits=None, name=None, process_set=None):
    if process_set is not None and process_set is not global_process_set:
        with _in_process_set(process_set):
            return alltoall(tensor, splits, name)
    return _alltoall_impl(tensor, splits, name)


def _alltoall_impl(tensor, splits=None, name=None):
    """Even alltoall in one kernel; with ``splits`` (rows of dim 0 sent to each rank, horovod semantics) the rows are
    padded to the largest split so the same even kernel moves them, and ``(output, received_splits)`` is returned."""
    import torch
    t = tensor.contiguous()
    e = _engine_for(tensor)
    if e is not None and not tensor.is_cuda:   # host tensors: ragged alltoallv in the engine, no padding
        sp = None if splits is None else [int(v) for v in (splits.tolist() if hasattr(splits, "tolist") else splits)]
        out, recv = e.alltoall_async(t, sp, name).wait()
        return out if splits is None else (out, recv)
    if splits is None:
        out = torch.empty_like(t)
        _comm().alltoall(t, out)
        return out
    n = size()
    sp = [int(v) for v in (splits.tolist() if hasattr(splits, "tolist") else splits)]
    if len(sp) != n or sum(sp) != t.shape[0] or min(sp) < 0:
        raise ValueError("alltoall: splits must have one non-negative entry per rank and sum to tensor.shape[0]")
    mine = torch.tensor(sp, dtype=torch.int32, device=t.device)
    all_splits = allgather(mine.view(1, n)).view(n, n)            # all_splits[src][dst]
    recv = [int(all_splits[src][rank()]) for src in range(n)]
    width = max(1, int(all_splits.max()))
    row = t.shape[1:]
    send = torch.zeros((n, width) + tuple(row), dtype=t.dtype, device=t.device)
    off = 0
    for dst in range(n):
        send[dst, :sp[dst]] = t[off:off + sp[dst]]
        off += sp[dst]
    got = torch.empty_like(send)
    _comm().alltoall(send, got)
    out = torch.cat([got[src, :recv[src]] for src in range(n)], dim=0) if sum(recv) else t.new_empty((0,) + tuple(row))
    return out, torch.tensor(recv, dtype=torch.int32)


def reducescatter(tensor, op=None, name=None, process_set=None):
    import torch
    if process_set is not None and process_set is not global_process_set:
        with _in_process_set(process_set):
            return reducescatter(tensor, op, name)
    t = tensor.contiguous()
    out = torch.empty((t.shape[0] // size(),) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    _comm().reduce_scatter(t, out, op=_op_name(op, None))
    return out


def alltoall_async(tensor, splits=None, name=None):
    """The exchange is issued in stream / call order and has completed (host) or been enqueued (device) when this returns."""
    return _Done(alltoall(tensor, splits, name))


def reducescatter_async(tensor, op=None, name=None):
    return _Done(reducescatter(tensor, op, name))


def grouped_reducescatter(tensors, op=None, name=None):
    return [reducescatter(t, op, f"{name}.{i}" if name else None) for i, t in enumerate(tensors)]


def grouped_reducescatter_async(tensors, op=None, name=None):
    return [reducescatter_async(t, op, f"{name}.{i}" if name else None) for i, t in enumerate(tensors)]


def is_homogeneous() -> bool:
    """Every node runs the same number of ranks: trivially true on one box."""
    return True


def _on_gpu() -> bool:
    return _comm().device != "cpu"


def _dev():
    return "cuda" if _on_gpu() else "cpu"


def barrier(process_set=None):
    import torch
    if process_set is not None and process_set is not global_process_set:
        with _in_process_set(process_set):
            return barrier()
    e = _state["engine"]
    if e is not None:
        e.barrier()
    else:
        _comm().barrier()
    if _on_gpu():
        torch.cuda.synchronize()


def join(device=-1) -> int:
    """Tell the other ranks this rank has run out of data: their allreduces keep completing (this rank contributes zeros)
    until every rank has joined. Returns the last rank that joined. Without the engine it degrades to a barrier."""
    e = _state["engine"]
    if e is not None:
        return e.join()
    barrier()
    return size() - 1


def synchronize(handle=None):
    """Wait for an ``*_async`` handle and return its output."""
    import torch
    if hasattr(handle, "wait"):
        out = handle.wait()
        if isinstance(handle, _Done) and _on_gpu():   # direct path: the work is queued on the current stream
            torch.cuda.current_stream().synchronize()
        return out
    if _on_gpu():
        torch.cuda.current_stream().synchronize()
    return handle


def poll(handle=None) -> bool:
    return handle.done() if hasattr(handle, "done") else True


def start_timeline(file_path: str, mark_cycles: bool = False) -> None:
    """Horovod Timeline (Chrome trace of every tensor's negotiation / fusion / reduction phases), written by rank 0;
    also enabled for the whole run by ``HOROVOD_TIMELINE=<path>``."""
    e = _state["engine"]
    if e is None:
        raise RuntimeError("the timeline is written by the background engine (not started; see B200MPI_HVD_ENGINE)")
    e.start_timeline(file_path)


def stop_timeline() -> None:
    e = _state["engine"]
    if e is not None:
        e.stop_timeline()


def engine_stats() -> dict:
    """Counters of the background engine: cycles, negotiated tensors, fused groups, cache hits / misses, stall warnings."""
    e = _state["engine"]
    return e.stats() if e is not None else {}


def broadcast_parameters(params, root_rank: int = 0) -> None:
    """K3 (tensorflow_mnist.py:143): state_dict / named_parameters / list of (name, tensor). Every tensor is submitted
    before the first wait, so with the engine the whole model is negotiated in one cycle."""
    import torch
    if isinstance(params, dict):
        items = sorted(params.items())
    else:
        items = list(params)
    handles = []
    for key, p in items:
        if isinstance(p, torch.Tensor) and (p.is_cuda or not _on_gpu()) and p.numel():
            handles.append(broadcast_async_(p.data, root_rank, name=f"broadcast_parameters.{key}"))
    for h in handles:
        h.wait()


def broadcast_object(obj, root_rank: int = 0, name=None):
    """Pickle on the root, broadcast, unpickle everywhere. The length travels as four 16-bit limbs in a float32 tensor
    (every limb is exact in fp32, any length up to 2^64 survives; a single float32 is only exact below 2^24 = 16 MiB)."""
    import pickle
    import torch
    payload = pickle.dumps(obj) if rank() == root_rank else b""
    ln0 = len(payload)
    n = torch.tensor([(ln0 >> (16 * k)) & 0xFFFF for k in range(4)], dtype=torch.float32, device=_dev())
    _comm().broadcast(n, root=root_rank)
    limbs = [int(v) for v in n.tolist()]
    ln = sum(v << (16 * k) for k, v in enumerate(limbs))
    if rank() == root_rank and ln != ln0:
        raise RuntimeError(f"broadcast_object: length {ln0} did not survive the broadcast ({ln})")
    buf = torch.zeros(ln + (-ln) % 2, dtype=torch.uint8, device=_dev())
    if rank() == root_rank:
        buf[:ln] = torch.frombuffer(bytearray(payload), dtype=torch.uint8).to(_dev())
    _comm().broadcast(buf, root=root_rank)
    return pickle.loads(bytes(buf[:ln].cpu().numpy()))


def allgather_object(obj, name=None) -> list:
    """One picklable object per rank -> list indexed by rank."""
    import pickle
    import torch
    payload = pickle.dumps(obj)
    lens = allgather(torch.tensor([len(payload)], dtype=torch.int64, device=_dev()))
    width = int(lens.max()) + (-int(lens.max())) % 2
    buf = torch.zeros(1, width, dtype=torch.uint8, device=_dev())
    buf[0, :len(payload)] = torch.frombuffer(bytearray(payload), dtype=torch.uint8).to(_dev())
    rows = allgather(buf).cpu()
    return [pickle.loads(bytes(rows[r, :int(lens[r])].numpy())) for r in range(size())]


def broadcast_optimizer_state(optimizer, root_rank: int = 0) -> None:
    """Rank `root_rank`'s optimizer state everywhere. The structure (param groups, scalar state) travels as one small
    pickle; state TENSORS (momentum buffers, Adam moments: hundreds of MB for a real model) are broadcast in place as
    tensors, never pickled."""
    import torch
    sd = optimizer.state_dict()
    tensors_root = []

    def strip(o):   # tensors -> placeholders (shape, dtype), in deterministic traversal order
        if isinstance(o, torch.Tensor):
            tensors_root.append(o)
            return ("__b200mpi_tensor__", len(tensors_root) - 1, tuple(o.shape), str(o.dtype).replace("torch.", ""), o.device.type)
        if isinstance(o, dict):
            return {k: strip(v) for k, v in o.items()}
        if isinstance(o, (list, tuple)):
            return type(o)(strip(v) for v in o)
        return o

    skeleton = strip(sd) if rank() == root_rank else None
    skeleton = broadcast_object(skeleton, root_rank)
    received = {}

    def fill(o):
        if isinstance(o, tuple) and len(o) == 5 and o[0] == "__b200mpi_tensor__":
            _, idx, shape, dt, devtype = o
            if rank() == root_rank:
                t = tensors_root[idx]
            else:
                t = torch.empty(shape, dtype=getattr(torch, dt), device=_dev() if devtype == "cuda" else "cpu")
            received[idx] = t
            return t
        if isinstance(o, dict):
            return {k: fill(v) for k, v in o.items()}
        if isinstance(o, (list, tuple)):
            return type(o)(fill(v) for v in o)
        return o

    full = fill(skeleton)
    for idx in sorted(received):
        t = received[idx]
        if t.numel() == 0:
            continue
        if (t.dtype in (torch.float32, torch.bfloat16, torch.float16) and t.is_contiguous() and t.dim() > 0
                and t.device.type == _dev()):
            broadcast_(t, root_rank, name=f"broadcast_optimizer_state.{idx}")
        else:   # step counters and other small non-float tensors
            v = broadcast_object(t.cpu() if rank() == root_rank else None, root_rank)
            if rank() != root_rank:
                t.copy_(v.to(t.device))
    if rank() != root_rank:
        optimizer.load_state_dict(full)


class Compression:
    class none:  # noqa: N801
        @staticmethod
        def compress(t): return t, None  # noqa: E704

        @staticmethod
        def decompress(t, ctx): return t  # noqa: E704

    class fp16:  # noqa: N801
        @staticmethod
        def compress(t): return t.half(), t.dtype  # noqa: E704

        @staticmethod
        def decompress(t, ctx): return t.to(ctx)  # noqa: E704


from .optimizer import DistributedOptimizer  # noqa: E402,F401

from .sync_batch_norm import SyncBatchNorm  # noqa: E402,F401
from . import elastic  # noqa: E402,F401
