"""Python face of the b200mpi collective runtime.

``Communicator`` wraps one ``b200mpi_comm_t``:

* ``Communicator.from_env()`` — one process per GPU (ranks found through the
  shm rendezvous; rank/world read from the launcher env, see
  ``mpi_operator_b200.launch.env`` and SURVEY.md Appendix B).
* ``Communicator.local(world)`` — ``world`` virtual ranks in this process on
  one device (every collective is ONE launch with ``gridDim.y == world``);
  used by unit tests, compute-sanitizer and ncu.

Symmetric windows are exposed as zero-copy ``torch`` tensors, so gradients can
be produced by autograd directly inside peer-visible memory.

Reference parity: the reference has no data plane; this replaces the
Horovod/NCCL calls its examples make (examples/v2beta1/horovod/
tensorflow_mnist.py:90-159).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Union

from . import _lib
from ._lib import (ALGO_AUTO, ALGO_NAMES, ALGO_NVLS, ALGO_ONESHOT, ALGO_TWOSHOT, BF16, F16, F32, MAX, MIN, SUM,
                   B200MPIError, check)

_ALGOS = {"auto": ALGO_AUTO, "oneshot": ALGO_ONESHOT, "twoshot": ALGO_TWOSHOT, "nvls": ALGO_NVLS}
_OPS = {"sum": SUM, "max": MAX, "min": MIN, "avg": SUM, "average": SUM}


def _torch():
    import torch
    return torch


def dtype_code(dtype) -> int:
    torch = _torch()
    if dtype == torch.float32:
        return F32
    if dtype == torch.bfloat16:
        return BF16
    if dtype == torch.float16:
        return F16
    raise B200MPIError(f"unsupported dtype {dtype} (float32, bfloat16, float16)")


class _CudaBlob:
    """Minimal ``__cuda_array_interface__`` carrier for a raw device pointer."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self._owner = owner
        self.__cuda_array_interface__ = {
            "shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None,
        }


def _stream_ptr(stream) -> int:
    torch = _torch()
    if stream is None:
        stream = torch.cuda.current_stream()
    return int(stream.cuda_stream)


def resolve_algo(algo: Union[str, int, None]) -> int:
    if algo is None:
        algo = os.environ.get("B200MPI_ALGO", "auto")
    if isinstance(algo, str):
        if algo not in _ALGOS:
            raise B200MPIError(f"unknown algorithm {algo!r} (auto|oneshot|twoshot|nvls)")
        return _ALGOS[algo]
    return int(algo)


class Window:
    """A symmetric allocation: same size on every rank, all peers mapped."""

    def __init__(self, comm: "Communicator", win: int, nbytes: int):
        self.comm, self.id, self.nbytes = comm, win, nbytes

    def ptr(self, rank: int = -1) -> int:
        return int(_lib.lib().b200mpi_window_ptr(self.comm._h, self.id, rank) or 0)

    @property
    def has_multicast(self) -> bool:
        return bool(_lib.lib().b200mpi_window_mc_ptr(self.comm._h, self.id))

    def tensor(self, dtype=None, rank: int = -1, offset: int = 0, numel: Optional[int] = None):
        """Zero-copy torch view of ``rank``'s copy (own copy by default)."""
        torch = _torch()
        dtype = dtype or torch.uint8
        esz = torch.empty((), dtype=dtype).element_size()
        if numel is None:
            numel = (self.nbytes - offset) // esz
        blob = _CudaBlob(self.ptr(rank) + offset, numel * esz, self)
        t = torch.as_tensor(blob, device=torch.device("cuda", self.comm.device))
        return t.view(dtype)

    def free(self) -> None:
        check(_lib.lib().b200mpi_window_free(self.comm._h, self.id), "window_free")


class Communicator:
    def __init__(self, handle: C.c_void_p, device: int):
        self._h = handle
        self.device = device
        L = _lib.lib()
        self.rank = L.b200mpi_comm_rank(handle)
        self.world = L.b200mpi_comm_world(handle)
        self.is_local = bool(L.b200mpi_comm_is_local(handle))
        self.has_multicast = bool(L.b200mpi_comm_has_multicast(handle))
        self._keep: list = []

    # ------------------------------------------------------------ creation --
    @classmethod
    def create(cls, rank: int, world: int, device: int, job_id: str, staging_bytes: int = 0, flags: int = 0):
        from . import affinity
        affinity.maybe_bind(device)      # B200MPI_BIND_TO=numa: run next to the GPU before the staging buffers are first touched
        h = C.c_void_p()
        check(_lib.lib().b200mpi_comm_init(C.byref(h), rank, world, device, job_id.encode(), staging_bytes, flags),
              "comm_init")
        c = cls(h, device)
        c._apply_tuning_file()
        if os.environ.get("B200MPI_STATS_DIR"):  # scripts that never call destroy() still report their counters
            import atexit
            import weakref
            ref = weakref.ref(c)
            atexit.register(lambda: ref() is not None and ref().dump_stats())
        return c

    def _apply_tuning_file(self) -> None:
        """Measured crossovers (benchmarks/autotune.py -> runtime/tuning.json; B200MPI_TUNING_FILE overrides).
        Explicit B200MPI_* env knobs win over the file."""
        import json
        path = os.environ.get("B200MPI_TUNING_FILE", os.path.join(os.path.dirname(os.path.abspath(__file__)), "tuning.json"))
        try:
            t = json.load(open(path))["by_world"].get(str(self.world))
        except (OSError, ValueError, KeyError):
            return
        if not t:
            return
        one = t.get("oneshot_max_bytes", -1) if "B200MPI_ONESHOT_MAX_BYTES" not in os.environ else -1
        nv = t.get("nvls_min_bytes", -1) if "B200MPI_NVLS_MIN_BYTES" not in os.environ else -1
        if nv == -1 and "nvls_min_bytes" in t and "B200MPI_NVLS_MIN_BYTES" not in os.environ:
            nv = (1 << 62)  # NVLS never wins at this world size
        self.set_tuning(oneshot_max_bytes=one if one > 0 else -1, nvls_min_bytes=nv)

    @classmethod
    def from_env(cls, device: Optional[int] = None, staging_bytes: int = 0, flags: int = 0):
        from ..launch.env import rank_info_from_env
        info = rank_info_from_env()
        if device is None:
            device = info.local_rank
        return cls.create(info.rank, info.world_size, device, info.job_id, staging_bytes, flags)

    @classmethod
    def local(cls, world: int, device: int = 0, staging_bytes: int = 0):
        h = C.c_void_p()
        check(_lib.lib().b200mpi_comm_init_local(C.byref(h), world, device, staging_bytes, 0), "comm_init_local")
        return cls(h, device)

    def destroy(self) -> None:
        if self._h:
            self.dump_stats()
            _lib.lib().b200mpi_comm_destroy(self._h)
            self._h = None

    # -------------------------------------------------------------- stats --
    def stats(self, native_only: bool = False) -> dict:
        """Counters by (op, algorithm) of every host-launched collective, plus whatever registered sources add
        (a DataParallelTrainer reports the kernels its CUDA graph replays). Feeds ``b200mpi_collective_*_total``
        on the operator's /metrics (SURVEY.md §5.5)."""
        import json
        L = _lib.lib()
        out = {"rank": self.rank, "world": self.world, "launches": 0, "ops": []}
        if self._h and hasattr(L, "b200mpi_comm_stats_json"):
            n = L.b200mpi_comm_stats_json(self._h, None, 0)
            buf = C.create_string_buffer(n + 1)
            L.b200mpi_comm_stats_json(self._h, buf, n + 1)
            out = json.loads(buf.value.decode())
        merged = {(o["op"], o["algo"]): dict(o) for o in out["ops"]}
        for src in ([] if native_only else getattr(self, "_stat_sources", [])):
            for o in src():
                m = merged.setdefault((o["op"], o["algo"]), {"op": o["op"], "algo": o["algo"], "calls": 0, "bytes": 0})
                m["calls"] += o["calls"]
                m["bytes"] += o["bytes"]
        out["ops"] = sorted(merged.values(), key=lambda o: (o["op"], o["algo"]))
        return out

    def add_stat_source(self, fn) -> None:
        if not hasattr(self, "_stat_sources"):
            self._stat_sources = []
        self._stat_sources.append(fn)

    def dump_stats(self, directory: Optional[str] = None) -> Optional[str]:
        """Write ``stats()`` to ``<dir>/stats-rank<r>-<pid>.json`` (dir defaults to $B200MPI_STATS_DIR, which the node
        agent sets per launcher pod and harvests when the pod finishes). No-op without a directory."""
        import json
        directory = directory or os.environ.get("B200MPI_STATS_DIR")
        if not directory or not self._h or self.is_local:
            return None
        try:
            os.makedirs(directory, exist_ok=True)
            path = os.path.join(directory, f"stats-rank{self.rank}-{os.getpid()}.json")
            with open(path + ".tmp", "w") as f:
                json.dump(self.stats(), f)
            os.replace(path + ".tmp", path)
            return path
        except OSError:
            return None

    # --------------------------------------------------------------- misc --
    @property
    def launch_count(self) -> int:
        return int(_lib.lib().b200mpi_comm_launch_count(self._h))

    def check_error(self) -> None:
        check(_lib.lib().b200mpi_comm_check_error(self._h), "collective watchdog")

    def host_barrier(self) -> None:
        check(_lib.lib().b200mpi_comm_host_barrier(self._h), "host_barrier")

    def host_allgather(self, payload: bytes) -> List[bytes]:
        n = len(payload)
        out = C.create_string_buffer(n * self.world)
        check(_lib.lib().b200mpi_comm_host_allgather(self._h, payload, out, n), "host_allgather")
        return [out.raw[i * n:(i + 1) * n] for i in range(self.world)]

    def set_tuning(self, oneshot_max_bytes: int = -1, nvls_min_bytes: int = -1, max_blocks: int = 0,
                   timeout_ms: int = 0) -> None:
        as_sz = lambda v: C.c_size_t(-1).value if v < 0 else v  # noqa: E731
        check(_lib.lib().b200mpi_set_tuning(self._h, as_sz(oneshot_max_bytes), as_sz(nvls_min_bytes), max_blocks,
                                            timeout_ms))

    def set_pipe(self, min_bytes: int = -1, lanes_nvls: int = 0, lanes_p2p: int = 0, depth: int = 0,
                 chunk_bytes: int = 0) -> None:
        """Pipelined user-pointer allreduce (``k_allreduce_pipe``): size threshold, lanes per mode, slots, chunk size."""
        check(_lib.lib().b200mpi_set_pipe(self._h, C.c_size_t(-1).value if min_bytes < 0 else min_bytes, lanes_nvls,
                                          lanes_p2p, depth, chunk_bytes))

    def set_reg(self, mode: int = -1, min_bytes: int = -1) -> None:
        """Lazy cudaIpc registration of user buffers: 0 never, 1 where the zero-copy P2P kernels win, 2 whenever possible."""
        check(_lib.lib().b200mpi_set_reg(self._h, mode, C.c_size_t(-1).value if min_bytes < 0 else min_bytes))

    def reg_stats(self) -> dict:
        a, b, c_ = C.c_uint64(), C.c_uint64(), C.c_uint64()
        _lib.lib().b200mpi_reg_stats(self._h, C.byref(a), C.byref(b), C.byref(c_))
        return {"zero_copy_calls": a.value, "handles_opened": b.value, "refused": c_.value}

    def get_tuning(self) -> dict:
        a, b, c_, d = C.c_size_t(), C.c_size_t(), C.c_int(), C.c_int()
        _lib.lib().b200mpi_get_tuning(self._h, C.byref(a), C.byref(b), C.byref(c_), C.byref(d))
        return {"oneshot_max_bytes": a.value, "nvls_min_bytes": b.value, "max_blocks": c_.value, "timeout_ms": d.value}

    def select_algo(self, nbytes: int, dtype_code_: int = F32, op: int = SUM, symmetric: bool = True) -> str:
        return ALGO_NAMES[_lib.lib().b200mpi_select_algo(self._h, nbytes, dtype_code_, op, int(symmetric))]

    def trace(self, on: bool = True) -> None:
        _lib.lib().b200mpi_trace_enable(self._h, int(on))

    def trace_dump(self, path: str) -> None:
        check(_lib.lib().b200mpi_trace_dump(self._h, path.encode()), "trace_dump")

    # ------------------------------------------------------------ windows --
    def alloc_window(self, nbytes: int) -> Window:
        w = C.c_int()
        check(_lib.lib().b200mpi_window_alloc(self._h, nbytes, C.byref(w)), "window_alloc")
        return Window(self, w.value, nbytes)

    # -------------------------------------------------------- collectives --
    def _ptrs(self, tensors):
        """real mode: one tensor -> its pointer; emulated: list of world tensors -> void*[world]."""
        if self.is_local:
            if not isinstance(tensors, (list, tuple)) or len(tensors) != self.world:
                raise B200MPIError("emulated communicator expects a list of `world` tensors")
            arr = (C.c_void_p * self.world)(*[t.data_ptr() for t in tensors])
            self._keep.append(arr)
            if len(self._keep) > 256:
                del self._keep[:128]
            return C.cast(arr, C.c_void_p), tensors[0]
        return C.c_void_p(tensors.data_ptr()), tensors

    @staticmethod
    def _scale(op: str, world: int, scale: Optional[float]) -> float:
        s = 1.0 if scale is None else float(scale)
        if op in ("avg", "average"):
            s /= world
        return s

    def allreduce_window(self, win: Window, offset: int, count: int, dtype, op: str = "sum",
                         scale: Optional[float] = None, algo=None, stream=None) -> None:
        """In-place allreduce of a 16-byte aligned window region."""
        check(_lib.lib().b200mpi_allreduce_sym(self._h, win.id, offset, count, dtype_code(dtype), _OPS[op],
                                               self._scale(op, self.world, scale), resolve_algo(algo),
                                               _stream_ptr(stream)), "allreduce_sym")

    def allgather_window(self, win: Window, offset: int, slice_bytes: int, stream=None) -> None:
        """Zero-copy allgather: the region is ``world`` slices of ``slice_bytes``; rank r's slice r (of its own copy) is
        delivered into slice r of every copy (one ``multimem.st`` per vector on NVLS)."""
        check(_lib.lib().b200mpi_allgather_sym(self._h, win.id, offset, slice_bytes, _stream_ptr(stream)), "allgather_sym")

    def reduce_scatter_window(self, win: Window, offset: int, slice_count: int, dtype, op: str = "sum",
                              scale: Optional[float] = None, out=None, stream=None) -> None:
        """Zero-copy reduce-scatter: slice r of every copy is reduced into rank r's ``out`` (slice-sized tensor) or, with
        ``out=None``, in place into slice r of rank r's own copy (``multimem.ld_reduce`` on NVLS)."""
        pout = self._ptrs(out)[0] if out is not None else None
        check(_lib.lib().b200mpi_reduce_scatter_sym(self._h, win.id, offset, slice_count, dtype_code(dtype), _OPS[op],
                                                    self._scale(op, self.world, scale), pout, _stream_ptr(stream)),
              "reduce_scatter_sym")

    def broadcast_window(self, win: Window, offset: int, nbytes: int, root: int = 0, stream=None) -> None:
        """Zero-copy broadcast of a window region from ``root``'s copy into every copy."""
        check(_lib.lib().b200mpi_broadcast_sym(self._h, win.id, offset, nbytes, root, _stream_ptr(stream)), "broadcast_sym")

    def allreduce(self, tensor, out=None, op: str = "sum", scale: Optional[float] = None, algo=None, stream=None):
        """Allreduce on arbitrary contiguous CUDA tensors (in place when ``out`` is None)."""
        out = tensor if out is None else out
        pin, t0 = self._ptrs(tensor)
        pout, _ = self._ptrs(out)
        if not t0.is_contiguous():
            raise B200MPIError("allreduce needs contiguous tensors")
        check(_lib.lib().b200mpi_allreduce(self._h, pin, pout, t0.numel(), dtype_code(t0.dtype), _OPS[op],
                                           self._scale(op, self.world, scale), resolve_algo(algo),
                                           _stream_ptr(stream)), "allreduce")
        return out

    def allreduce_sgd_window(self, grad_win: Window, grad_off: int, param_win: Window, param_off: int, momentum,
                             count: int, grad_dtype, lr: float, momentum_coef: float = 0.0, weight_decay: float = 0.0,
                             nesterov: bool = False, first_step: bool = False, scale: Optional[float] = None,
                             lowp_win: Optional[Window] = None, lowp_off: int = 0, algo=None, stream=None,
                             group_map=None, group_hyper=None, ema=None, ema_sched=None) -> None:
        """Fused gradient-average + SGD step; see b200mpi_allreduce_sgd_sym.

        Parameter groups (fp32 gradients only): ``group_map`` is a CUDA uint8 tensor of ``count // 4`` entries, the group of
        each 4-element vector of this region (already offset to it), and ``group_hyper`` a contiguous CUDA float32 ``[G, 3]``
        tensor of ``{lr, momentum, weight_decay}`` rows, read by the kernel at run time, which then replaces ``lr``,
        ``momentum_coef``, ``weight_decay`` and ``set_hyper``'s tensor. Every map entry must be ``< G``; the kernel does not
        check it. On an emulated communicator one map and one table serve every rank.

        Weight average (fp32 gradients only; see b200mpi_allreduce_sgd_sym_ema): ``ema`` is this rank's float32 shard of
        ``slice_elems(count)`` elements, laid out like ``momentum`` (emulated: a list of ``world``), and ``ema_sched`` a
        contiguous float64 CUDA tensor ``[decay, updates]`` read at run time; the two go together."""
        pm, _ = self._ptrs(momentum)
        s = (1.0 / self.world) if scale is None else float(scale)
        pe = self._ema_ptrs("allreduce_sgd_window", count, grad_dtype, ema, ema_sched)
        if pe is not None:
            check(_lib.lib().b200mpi_allreduce_sgd_sym_ema(
                self._h, grad_win.id, grad_off, param_win.id, param_off, lowp_win.id if lowp_win else -1, lowp_off, pm,
                count, dtype_code(grad_dtype), s, lr, momentum_coef, weight_decay, int(nesterov), int(first_step),
                resolve_algo(algo), _stream_ptr(stream),
                *self._group_ptrs("allreduce_sgd_window", count, grad_dtype, group_map, group_hyper), *pe),
                "allreduce_sgd_sym_ema")
            return
        if group_map is not None or group_hyper is not None:
            check(_lib.lib().b200mpi_allreduce_sgd_sym_groups(
                self._h, grad_win.id, grad_off, param_win.id, param_off, lowp_win.id if lowp_win else -1, lowp_off, pm,
                count, dtype_code(grad_dtype), s, lr, momentum_coef, weight_decay, int(nesterov), int(first_step),
                resolve_algo(algo), _stream_ptr(stream),
                *self._group_ptrs("allreduce_sgd_window", count, grad_dtype, group_map, group_hyper)),
                "allreduce_sgd_sym_groups")
            return
        check(_lib.lib().b200mpi_allreduce_sgd_sym(
            self._h, grad_win.id, grad_off, param_win.id, param_off, lowp_win.id if lowp_win else -1, lowp_off, pm,
            count, dtype_code(grad_dtype), s, lr, momentum_coef, weight_decay, int(nesterov), int(first_step),
            resolve_algo(algo), _stream_ptr(stream)), "allreduce_sgd_sym")

    def _group_ptrs(self, name: str, count: int, grad_dtype, group_map, group_hyper) -> tuple:
        """Checked (map, table, rows) of the grouped entry points: all null without parameter groups."""
        if group_map is None and group_hyper is None:
            return None, None, 0
        torch = _torch()
        dev = torch.device("cuda", self.device)
        if group_map is None or group_hyper is None:
            raise B200MPIError(f"{name}: group_map and group_hyper go together")
        if grad_dtype != torch.float32:
            raise B200MPIError(f"{name}: parameter groups need float32 gradients")
        if not (group_map.device == dev and group_map.dtype == torch.uint8 and group_map.is_contiguous()
                and group_map.numel() == count // 4):
            raise B200MPIError(f"{name}: group_map must be a contiguous uint8 tensor of {count // 4} entries on {dev}")
        if not (group_hyper.device == dev and group_hyper.dtype == torch.float32 and group_hyper.is_contiguous()
                and group_hyper.dim() == 2 and group_hyper.shape[1] == 3 and 1 <= group_hyper.shape[0] <= 256):
            raise B200MPIError(f"{name}: group_hyper must be a contiguous float32 [G, 3] tensor on {dev}, 1 <= G <= 256")
        return group_map.data_ptr(), group_hyper.data_ptr(), int(group_hyper.shape[0])

    def _ema_ptrs(self, name: str, count: int, grad_dtype, ema, ema_sched) -> Optional[tuple]:
        """Checked (ema, ema_sched) pointers of the ``_ema`` entry points, or None when neither is given."""
        if ema is None and ema_sched is None:
            return None
        torch = _torch()
        dev = torch.device("cuda", self.device)
        if ema is None or ema_sched is None:
            raise B200MPIError(f"{name}: ema and ema_sched go together")
        if grad_dtype != torch.float32:
            raise B200MPIError(f"{name}: the weight average needs float32 gradients")
        n = self.slice_elems(count, torch.float32)
        shards = ema if isinstance(ema, (list, tuple)) else [ema]
        if any(not (t.device == dev and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == n) for t in shards):
            raise B200MPIError(f"{name}: ema must be contiguous float32 tensors of {n} elements on {dev}")
        if not (ema_sched.device == dev and ema_sched.dtype == torch.float64 and ema_sched.is_contiguous()
                and ema_sched.numel() == 2):
            raise B200MPIError(f"{name}: ema_sched must be a contiguous float64 tensor of 2 elements on {dev}")
        return self._ptrs(ema)[0], ema_sched.data_ptr()

    def lars_scratch_bytes(self, count: int, num_params: int) -> int:
        """Bytes of the per-rank scratch ``allreduce_lars_window`` needs for a region of ``count`` fp32 elements."""
        return int(_lib.lib().b200mpi_lars_scratch_bytes(count, self.world, num_params))

    def allreduce_lars_window(self, grad_win: Window, grad_off: int, param_win: Window, param_off: int, momentum,
                              count: int, grad_dtype, *, group_hyper, param_map, param_table, board_win: Window,
                              board_off: int, scratch, trust_coefficient: float, nesterov: bool = False,
                              first_step: bool = False, scale: Optional[float] = None, lowp_win: Optional[Window] = None,
                              lowp_off: int = 0, algo=None, stream=None, trust_out=None, ema=None,
                              ema_sched=None) -> None:
        """Fused gradient-average + LARS step; see b200mpi_allreduce_lars_sym. Two launches on ``stream``.

        ``param_map`` is a CUDA uint16 tensor of ``count // 4`` entries, the bucket-local parameter of each 4-element vector
        (non-decreasing; vectors past the last parameter hold ``P``), ``param_table`` a contiguous CUDA uint8 ``[P, 2]``
        tensor of ``{group, lars}`` rows and ``group_hyper`` the ``[G, 3]`` table of ``allreduce_sgd_window``. ``board_win``
        holds ``P * world`` float pairs at ``board_off``. ``scratch`` is this rank's zero-filled CUDA uint8 tensor of at
        least ``lars_scratch_bytes(count, P)`` bytes and ``trust_out`` an optional float32 ``[P]`` tensor that receives the
        trust ratios (on an emulated communicator: lists of ``world`` tensors, one per rank). ``ema`` / ``ema_sched`` add the
        weight average of ``allreduce_sgd_window``."""
        torch = _torch()
        if grad_dtype != torch.float32:
            raise B200MPIError("allreduce_lars_window: LARS needs float32 gradients")
        dev = torch.device("cuda", self.device)
        if not (param_map.device == dev and param_map.dtype == torch.uint16 and param_map.is_contiguous()
                and param_map.numel() == count // 4):
            raise B200MPIError(f"allreduce_lars_window: param_map must be a contiguous uint16 tensor of {count // 4} entries on {dev}")
        if not (param_table.device == dev and param_table.dtype == torch.uint8 and param_table.is_contiguous()
                and param_table.dim() == 2 and param_table.shape[1] == 2 and param_table.shape[0] >= 1):
            raise B200MPIError(f"allreduce_lars_window: param_table must be a contiguous uint8 [P, 2] tensor on {dev}")
        if not (group_hyper.device == dev and group_hyper.dtype == torch.float32 and group_hyper.is_contiguous()
                and group_hyper.dim() == 2 and group_hyper.shape[1] == 3 and 1 <= group_hyper.shape[0] <= 256):
            raise B200MPIError(f"allreduce_lars_window: group_hyper must be a contiguous float32 [G, 3] tensor on {dev}, 1 <= G <= 256")
        P = int(param_table.shape[0])
        scr = scratch if isinstance(scratch, (list, tuple)) else [scratch]
        if any(not (s.device == dev and s.dtype == torch.uint8 and s.is_contiguous()) for s in scr):
            raise B200MPIError(f"allreduce_lars_window: scratch must be contiguous uint8 tensors on {dev}")
        if trust_out is not None:
            outs = trust_out if isinstance(trust_out, (list, tuple)) else [trust_out]
            if any(not (t.device == dev and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == P) for t in outs):
                raise B200MPIError(f"allreduce_lars_window: trust_out must be contiguous float32 tensors of {P} entries on {dev}")
        pm, _ = self._ptrs(momentum)
        ps, _ = self._ptrs(scratch)
        pt = self._ptrs(trust_out)[0] if trust_out is not None else None
        s = (1.0 / self.world) if scale is None else float(scale)
        pe = self._ema_ptrs("allreduce_lars_window", count, grad_dtype, ema, ema_sched)
        if pe is not None:
            check(_lib.lib().b200mpi_allreduce_lars_sym_ema(
                self._h, grad_win.id, grad_off, param_win.id, param_off, lowp_win.id if lowp_win else -1, lowp_off, pm,
                count, dtype_code(grad_dtype), s, int(nesterov), int(first_step), resolve_algo(algo), _stream_ptr(stream),
                group_hyper.data_ptr(), int(group_hyper.shape[0]), param_map.data_ptr(), param_table.data_ptr(), P,
                board_win.id, board_off, ps, min(t.numel() for t in scr), float(trust_coefficient), pt, *pe),
                "allreduce_lars_sym_ema")
            return
        check(_lib.lib().b200mpi_allreduce_lars_sym(
            self._h, grad_win.id, grad_off, param_win.id, param_off, lowp_win.id if lowp_win else -1, lowp_off, pm, count,
            dtype_code(grad_dtype), s, int(nesterov), int(first_step), resolve_algo(algo), _stream_ptr(stream),
            group_hyper.data_ptr(), int(group_hyper.shape[0]), param_map.data_ptr(), param_table.data_ptr(), P,
            board_win.id, board_off, ps, min(t.numel() for t in scr), float(trust_coefficient), pt),
            "allreduce_lars_sym")

    # ------------------------------------------------------ point-to-point --
    @property
    def has_p2p(self) -> bool:
        L = _lib.lib()
        return bool(hasattr(L, "b200mpi_comm_has_p2p") and L.b200mpi_comm_has_p2p(self._h))

    def p2p_batch(self, ops, stream=None) -> None:
        """EXPERIMENTAL (needs B200MPI_P2P=1 at creation). ``ops``: list of ``("send" | "recv", tensor, peer)``; the whole
        batch runs as one kernel with one CTA per operation, so a rank may send to and receive from the same peers in one
        call without deadlocking (the ncclGroupStart/End pattern)."""

        class _Op(C.Structure):
            _fields_ = [("send", C.c_void_p), ("recv", C.c_void_p), ("bytes", C.c_size_t), ("peer", C.c_int), ("is_send", C.c_int)]
        arr = (_Op * len(ops))()
        for k, (kind, t, peer) in enumerate(ops):
            if kind not in ("send", "recv") or not t.is_contiguous() or not t.is_cuda:
                raise B200MPIError("p2p_batch: ('send'|'recv', contiguous CUDA tensor, peer)")
            nbytes = t.numel() * t.element_size()
            arr[k] = _Op(t.data_ptr() if kind == "send" else None, t.data_ptr() if kind == "recv" else None, nbytes, int(peer),
                         1 if kind == "send" else 0)
        check(_lib.lib().b200mpi_p2p_batch(self._h, C.cast(arr, C.c_void_p), len(ops), _stream_ptr(stream)), "p2p_batch")

    def send(self, tensor, peer: int, stream=None) -> None:
        self.p2p_batch([("send", tensor, peer)], stream)

    def recv(self, tensor, peer: int, stream=None) -> None:
        self.p2p_batch([("recv", tensor, peer)], stream)

    def set_hyper(self, tensor) -> None:
        """Device tensor {lr, momentum, weight_decay} read by the fused SGD kernels (None: by-value)."""
        self._hyper = tensor
        check(_lib.lib().b200mpi_set_hyper_ptr(self._h, tensor.data_ptr() if tensor is not None else None))

    def lr_schedule(self, table, form: int, num_boundaries: int, step, base, hyper, group_hyper=None, stream=None) -> None:
        """One launch of ``k_lr_schedule`` on ``stream``; see b200mpi_lr_schedule. ``table`` is the float64 table of
        ``LRSchedule.table()`` on the device, ``step`` an int64 counter of one element, ``base`` the float64 base rates
        ``[G]``, ``hyper`` the ``set_hyper`` tensor and ``group_hyper`` the optional float32 ``[G, 3]`` group table; all
        contiguous CUDA tensors on this communicator's device. Writes the rates of step ``step`` and advances it by one."""
        torch = _torch()
        dev = torch.device("cuda", self.device)

        def ok(t, dtype, n=None):
            return t.device == dev and t.dtype == dtype and t.is_contiguous() and (n is None or t.numel() == n)
        if not ok(table, torch.float64):
            raise B200MPIError(f"lr_schedule: table must be a contiguous float64 tensor on {dev}")
        if not ok(step, torch.int64, 1):
            raise B200MPIError(f"lr_schedule: step must be a contiguous int64 tensor of 1 element on {dev}")
        if not (ok(base, torch.float64) and base.dim() == 1 and 1 <= base.numel() <= 256):
            raise B200MPIError(f"lr_schedule: base must be a contiguous float64 [G] tensor on {dev}, 1 <= G <= 256")
        G = base.numel()
        if not (ok(hyper, torch.float32) and hyper.numel() >= 1):
            raise B200MPIError(f"lr_schedule: hyper must be a contiguous float32 tensor on {dev}")
        if group_hyper is not None and not (ok(group_hyper, torch.float32, 3 * G) and group_hyper.dim() == 2):
            raise B200MPIError(f"lr_schedule: group_hyper must be a contiguous float32 [{G}, 3] tensor on {dev}")
        if table.numel() < 1 + (2 * num_boundaries + 1 if form == 1 else 3 if form in (2, 3) else 0):
            raise B200MPIError("lr_schedule: table shorter than its form and boundary count need")
        check(_lib.lib().b200mpi_lr_schedule(self._h, table.data_ptr(), int(form), int(num_boundaries), step.data_ptr(),
                                             base.data_ptr(), G, hyper.data_ptr(),
                                             group_hyper.data_ptr() if group_hyper is not None else None,
                                             _stream_ptr(stream)), "lr_schedule")

    def slice_elems(self, count: int, dtype) -> int:
        return int(_lib.lib().b200mpi_slice_elems(count, self.world, dtype_code(dtype)))

    def broadcast(self, tensor, root: int = 0, stream=None):
        p, t0 = self._ptrs(tensor)
        check(_lib.lib().b200mpi_broadcast_bytes(self._h, p, t0.numel() * t0.element_size(), root,
                                                 _stream_ptr(stream)), "broadcast")
        return tensor

    def allgather(self, tensor, out, stream=None):
        pin, t0 = self._ptrs(tensor)
        pout, _ = self._ptrs(out)
        nbytes = t0.numel() * t0.element_size()
        if nbytes % 2:
            raise B200MPIError("allgather payload must be an even number of bytes")
        # the kernel is byte-wise; express the payload in 2-byte units
        check(_lib.lib().b200mpi_allgather(self._h, pin, pout, nbytes // 2, BF16, _stream_ptr(stream)), "allgather")
        return out

    def adasum_max_bytes(self, dtype) -> int:
        """Largest tensor (bytes) the one-kernel Adasum takes on this communicator; 0 when it cannot run at all (world
        not a power of two, dtype other than f32 / bf16 / f16, staging window too small)."""
        if self.world < 2 or self.world & (self.world - 1):
            return 0
        try:
            code = dtype_code(dtype)
        except Exception:
            return 0
        if code not in (F32, BF16, F16):
            return 0
        return int(_lib.lib().b200mpi_adasum_max_bytes(self._h, code))

    def adasum(self, tensor, out=None, stream=None):
        """Adasum allreduce (Horovod ``op=hvd.Adasum``) in ONE kernel (csrc/kernels/adasum.cu): slice-parallel
        distance-doubling tree over peer memory, dot products exchanged through a board in the staging window.
        Raises B200MPIError when ``adasum_max_bytes`` says the tensor does not fit; ``hvd/adasum.py`` then gathers
        and folds the tree with torch ops."""
        out = tensor if out is None else out
        pin, t0 = self._ptrs(tensor)
        pout, _ = self._ptrs(out)
        check(_lib.lib().b200mpi_adasum(self._h, pin, pout, t0.numel(), dtype_code(t0.dtype), _stream_ptr(stream)), "adasum")
        return out

    def reduce_scatter(self, tensor, out, op: str = "sum", scale: Optional[float] = None, stream=None):
        pin, _ = self._ptrs(tensor)
        pout, o0 = self._ptrs(out)
        check(_lib.lib().b200mpi_reduce_scatter(self._h, pin, pout, o0.numel(), dtype_code(o0.dtype), _OPS[op],
                                                self._scale(op, self.world, scale), _stream_ptr(stream)),
              "reduce_scatter")
        return out

    def reduce(self, tensor, out=None, root: int = 0, op: str = "sum", scale: Optional[float] = None, stream=None):
        out = tensor if out is None else out
        pin, t0 = self._ptrs(tensor)
        pout, _ = self._ptrs(out)
        check(_lib.lib().b200mpi_reduce(self._h, pin, pout, t0.numel(), dtype_code(t0.dtype), _OPS[op],
                                        self._scale(op, self.world, scale), root, _stream_ptr(stream)), "reduce")
        return out

    def alltoall(self, tensor, out, stream=None):
        pin, t0 = self._ptrs(tensor)
        pout, _ = self._ptrs(out)
        per = t0.numel() // self.world
        check(_lib.lib().b200mpi_alltoall(self._h, pin, pout, per, dtype_code(t0.dtype), _stream_ptr(stream)),
              "alltoall")
        return out

    def barrier(self, stream=None) -> None:
        check(_lib.lib().b200mpi_barrier(self._h, _stream_ptr(stream)), "barrier")


def scale_cast(src, dst, scale: float = 1.0, stream=None):
    """dst = cast(src * scale) in one kernel (used by the bucketing engine)."""
    check(_lib.lib().b200mpi_scale_cast(src.data_ptr(), dtype_code(src.dtype), dst.data_ptr(), dtype_code(dst.dtype),
                                        src.numel(), scale, _stream_ptr(stream)), "scale_cast")
    return dst
