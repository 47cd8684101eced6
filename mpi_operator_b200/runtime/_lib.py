"""ctypes binding of libb200mpi.so (csrc/include/b200mpi.h).

The library is built in-tree by ``make`` / ``__graft_entry__.build()`` into
``mpi_operator_b200/lib``.  Loading is explicit and loud: on a GPU box a missing
library is an error, never a silent PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

_PKG = Path(__file__).resolve().parent.parent
_ROOT = _PKG.parent
LIB_PATH = _PKG / "lib" / "libb200mpi.so"

F32, BF16, F16 = 0, 1, 2
SUM, MAX, MIN = 0, 1, 2
ALGO_AUTO, ALGO_ONESHOT, ALGO_TWOSHOT, ALGO_NVLS = 0, 1, 2, 3
ALGO_NAMES = {0: "auto", 1: "oneshot", 2: "twoshot", 3: "nvls"}
FLAG_NO_MULTICAST, FLAG_FORCE_IPC, FLAG_NO_PIPE = 1, 2, 4

_lib = None


class B200MPIError(RuntimeError):
    pass


def build(force: bool = False) -> Path:
    """Compile libb200mpi.so for sm_90a with nvcc (no GPU needed)."""
    if LIB_PATH.exists() and not force:
        srcs = list((_ROOT / "csrc").rglob("*.cu")) + list((_ROOT / "csrc").rglob("*.cc")) + \
            list((_ROOT / "csrc").rglob("*.h")) + list((_ROOT / "csrc").rglob("*.cuh"))
        if srcs and max(s.stat().st_mtime for s in srcs) <= LIB_PATH.stat().st_mtime:
            return LIB_PATH
    subprocess.run(["make", "-C", str(_ROOT), "all"], check=True)
    return LIB_PATH


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        if os.environ.get("B200MPI_NO_AUTOBUILD"):
            raise B200MPIError(f"{LIB_PATH} is missing; run `make` (or __graft_entry__.build())")
        build()
    # When the NCCL-ABI shim is LD_PRELOADed (the node agent injects it into every rank) it already contains the whole
    # runtime - same sources, same symbols. Loading libb200mpi.so next to it would put two copies of every kernel stub and
    # every exported helper into one process, with calls between them resolved to whichever copy comes first: use the
    # preloaded one as THE runtime instead.
    path = str(LIB_PATH)
    for pre in os.environ.get("LD_PRELOAD", "").replace(" ", ":").split(":"):
        if pre.endswith("libb200mpi_nccl.so") and os.path.exists(pre):
            path = pre
            break
    L = C.CDLL(path, mode=C.RTLD_GLOBAL)
    vp, sz, i, u, f = C.c_void_p, C.c_size_t, C.c_int, C.c_uint, C.c_float
    L.b200mpi_last_error.restype = C.c_char_p
    L.b200mpi_version.restype = C.c_char_p
    L.b200mpi_comm_init.argtypes = [C.POINTER(vp), i, i, i, C.c_char_p, sz, u]
    L.b200mpi_comm_init_local.argtypes = [C.POINTER(vp), i, i, sz, u]
    L.b200mpi_comm_destroy.argtypes = [vp]
    for name in ("rank", "world", "is_local", "has_multicast", "host_barrier", "check_error"):
        getattr(L, f"b200mpi_comm_{name}").argtypes = [vp]
    L.b200mpi_comm_host_allgather.argtypes = [vp, vp, vp, sz]
    L.b200mpi_comm_launch_count.argtypes = [vp]
    L.b200mpi_comm_launch_count.restype = C.c_uint64
    L.b200mpi_window_alloc.argtypes = [vp, sz, C.POINTER(i)]
    L.b200mpi_window_free.argtypes = [vp, i]
    L.b200mpi_window_ptr.argtypes = [vp, i, i]
    L.b200mpi_window_ptr.restype = vp
    L.b200mpi_window_mc_ptr.argtypes = [vp, i]
    L.b200mpi_window_mc_ptr.restype = vp
    L.b200mpi_window_size.argtypes = [vp, i]
    L.b200mpi_window_size.restype = sz
    L.b200mpi_allreduce_sym.argtypes = [vp, i, sz, sz, i, i, f, i, vp]
    L.b200mpi_allreduce.argtypes = [vp, vp, vp, sz, i, i, f, i, vp]
    L.b200mpi_allreduce_sgd_sym.argtypes = [vp, i, sz, i, sz, i, sz, vp, sz, i, f, f, f, f, i, i, i, vp]
    L.b200mpi_slice_elems.argtypes = [sz, i, i]
    L.b200mpi_slice_elems.restype = sz
    L.b200mpi_set_hyper_ptr.argtypes = [vp, vp]
    L.b200mpi_broadcast.argtypes = [vp, vp, sz, i, i, vp]
    L.b200mpi_broadcast_bytes.argtypes = [vp, vp, sz, i, vp]
    L.b200mpi_allgather.argtypes = [vp, vp, vp, sz, i, vp]
    L.b200mpi_reduce_scatter.argtypes = [vp, vp, vp, sz, i, i, f, vp]
    L.b200mpi_adasum.argtypes = [vp, vp, vp, sz, i, vp]
    L.b200mpi_adasum_max_bytes.argtypes = [vp, i]
    L.b200mpi_adasum_max_bytes.restype = sz
    L.b200mpi_reduce.argtypes = [vp, vp, vp, sz, i, i, f, i, vp]
    L.b200mpi_alltoall.argtypes = [vp, vp, vp, sz, i, vp]
    L.b200mpi_barrier.argtypes = [vp, vp]
    L.b200mpi_scale_cast.argtypes = [vp, i, vp, i, sz, f, vp]
    L.b200mpi_bn_workspace_floats.argtypes = [i]
    L.b200mpi_bn_workspace_floats.restype = sz
    L.b200mpi_bn_supported.argtypes = [C.c_longlong, i]
    L.b200mpi_bn_act_fwd.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_longlong, i, f, f, i, vp]
    if hasattr(L, "b200mpi_bn_act_fwd_prestats"):
        L.b200mpi_bn_act_fwd_prestats.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i, C.c_longlong, i, f, f, i, vp]
    L.b200mpi_bn_act_bwd.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_longlong, i, i, vp]
    L.b200mpi_set_tuning.argtypes = [vp, sz, sz, i, i]
    L.b200mpi_get_tuning.argtypes = [vp, C.POINTER(sz), C.POINTER(sz), C.POINTER(i), C.POINTER(i)]
    L.b200mpi_select_algo.argtypes = [vp, sz, i, i, i]
    L.b200mpi_set_pipe.argtypes = [vp, sz, i, i, i, sz]
    L.b200mpi_set_reg.argtypes = [vp, i, sz]
    L.b200mpi_reg_stats.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.b200mpi_allgather_sym.argtypes = [vp, i, sz, sz, vp]
    L.b200mpi_reduce_scatter_sym.argtypes = [vp, i, sz, sz, i, i, f, vp, vp]
    L.b200mpi_broadcast_sym.argtypes = [vp, i, sz, sz, i, vp]
    if hasattr(L, "b200mpi_p2p_batch"):  # experimental point-to-point (csrc/kernels/p2p.cu)
        L.b200mpi_p2p_batch.argtypes = [vp, vp, i, vp]
        L.b200mpi_comm_has_p2p.argtypes = [vp]
    if hasattr(L, "b200mpi_comm_stats_json"):  # absent only in a stale build
        L.b200mpi_comm_stats_json.argtypes = [vp, C.c_char_p, C.c_size_t]
        L.b200mpi_comm_stats_json.restype = C.c_int
    L.b200mpi_trace_enable.argtypes = [vp, i]
    L.b200mpi_trace_dump.argtypes = [vp, C.c_char_p]
    _lib = L
    return L


def check(rc: int, what: str = "b200mpi") -> None:
    if rc != 0:
        msg = lib().b200mpi_last_error()
        raise B200MPIError(f"{what} failed ({rc}): {msg.decode() if msg else '?'}")
