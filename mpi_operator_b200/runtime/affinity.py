"""CPU affinity next to a rank's GPU, for ranks that were not started by the in-tree ``mpirun`` (torchrun, a notebook, srun).

On an 8-GPU HGX board GPUs 0-3 and 4-7 hang off different sockets. A rank whose host thread runs on the far socket first-touches
its pinned staging buffers in far memory, and every H2D copy of the input batch then crosses the socket interconnect. Open MPI's
answer is ``--bind-to numa`` (the reference's command lines say ``-bind-to none``, examples/v2beta1/tensorflow-benchmarks/
tensorflow-benchmarks.yaml:23-24, which stays the default here); ``csrc/spawner/mpirun.cc`` implements that flag with GPU locality,
and this module gives the same placement to a process that is already running: ``B200MPI_BIND_TO=numa`` makes
``Communicator.create`` call :func:`bind_near_gpu` before anything is allocated. Ranks that ``mpirun`` already bound
(``B200MPI_BOUND_CPUS`` in the environment) are left alone.

Everything is read from sysfs (``/sys/bus/pci/devices/<bus id>/numa_node``, ``/sys/devices/system/node/node<N>/cpulist``);
``B200MPI_SYSFS_ROOT`` re-roots the paths (tests). Nothing here needs CUDA: the bus id comes from torch's device properties when
a CUDA context is around, from the ordering of ``/proc/driver/nvidia/gpus`` (PCI bus order, what ``nvidia-smi`` and
``CUDA_DEVICE_ORDER=PCI_BUS_ID`` use) otherwise.
"""
from __future__ import annotations

import os
from typing import List, Optional, Set


def _root() -> str:
    return os.environ.get("B200MPI_SYSFS_ROOT", "")


def parse_cpulist(text: str) -> List[int]:
    out: List[int] = []
    for tok in text.strip().split(","):
        if not tok:
            continue
        a, _, b = tok.partition("-")
        try:
            lo, hi = int(a), int(b or a)
        except ValueError:
            continue
        out.extend(range(lo, hi + 1))
    return out


def format_cpulist(cpus) -> str:
    cpus, out, k = sorted(cpus), [], 0
    while k < len(cpus):
        e = k
        while e + 1 < len(cpus) and cpus[e + 1] == cpus[e] + 1:
            e += 1
        out.append(str(cpus[k]) if e == k else f"{cpus[k]}-{cpus[e]}")
        k = e + 1
    return ",".join(out)


def physical_gpu_index(device: int) -> int:
    """CUDA ordinal -> index on the box (CUDA_VISIBLE_DEVICES with numeric entries re-numbers the devices)."""
    cvd = os.environ.get("CUDA_VISIBLE_DEVICES", "")
    ids = [t.strip() for t in cvd.split(",") if t.strip()]
    if 0 <= device < len(ids) and ids[device].isdigit():
        return int(ids[device])
    return device


def gpu_bus_id(device: int) -> Optional[str]:
    try:
        import torch
        if torch.cuda.is_available() and not _root():
            p = torch.cuda.get_device_properties(device)
            return f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
    except Exception:  # noqa: BLE001  (older torch without the pci_* properties, no driver)
        pass
    try:
        bus = sorted(os.listdir(_root() + "/proc/driver/nvidia/gpus"))
    except OSError:
        return None
    idx = physical_gpu_index(device)
    return bus[idx].lower() if 0 <= idx < len(bus) else None


def gpu_numa_node(device: int) -> Optional[int]:
    bus = gpu_bus_id(device)
    if bus is None:
        return None
    try:
        node = int(open(f"{_root()}/sys/bus/pci/devices/{bus}/numa_node").read().strip())
    except (OSError, ValueError):
        return None
    return node if node >= 0 else None          # -1: the platform does not say (single-socket boxes, some VMs)


def numa_cpus(node: int) -> Set[int]:
    try:
        return set(parse_cpulist(open(f"{_root()}/sys/devices/system/node/node{node}/cpulist").read()))
    except OSError:
        return set()


def bind_near_gpu(device: int) -> Optional[dict]:
    """Restrict the calling thread - and every thread or child it starts afterwards; call it before thread pools start - to the
    CPUs of the GPU's NUMA node that it may already run on. Returns ``{"numa": n, "cpus": "0-55"}`` or None when nothing was
    changed (no NUMA information, the intersection is empty, or the kernel refused)."""
    node = gpu_numa_node(device)
    if node is None:
        return None
    allowed = os.sched_getaffinity(0)
    cpus = numa_cpus(node) & allowed
    if not cpus or cpus == allowed:
        return None
    try:
        os.sched_setaffinity(0, cpus)
    except OSError:
        return None
    info = {"numa": node, "cpus": format_cpulist(cpus)}
    os.environ["B200MPI_BOUND_CPUS"], os.environ["B200MPI_BOUND_NUMA"] = info["cpus"], str(node)
    return info


def maybe_bind(device: int) -> Optional[dict]:
    """The hook ``Communicator.create`` calls: binds only when asked to (``B200MPI_BIND_TO=numa|socket``) and only once."""
    if os.environ.get("B200MPI_BIND_TO", "none").split(":")[0] not in ("numa", "socket", "package"):
        return None
    if os.environ.get("B200MPI_BOUND_CPUS"):
        return None
    return bind_near_gpu(device)
