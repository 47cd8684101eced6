"""GPU / NVLink topology discovery.

The reference asks the Kubernetes API server where capacity is; a single-box
daemon asks the hardware (BASELINE.json north-star).  Discovery order: NVML
(``pynvml`` from nvidia-ml-py: device list, UUIDs, NVLink P2P status), then
``torch.cuda``, then ``B200MPI_FAKE_GPUS=N`` for tests.  On an HGX H100 board every
pair is an NVSwitch peer, so any k-of-8 placement is bandwidth-equivalent; we
still record per-pair P2P capability and refuse non-peer placements.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional


@dataclass
class GPU:
    index: int
    uuid: str = ""
    name: str = ""
    memory_bytes: int = 0
    nvlink_peers: List[int] = field(default_factory=list)
    pci_bus_id: str = ""
    numa_node: Optional[int] = None     # the socket whose PCIe root the GPU hangs off (sysfs); None = the platform does not say


@dataclass
class Topology:
    gpus: List[GPU] = field(default_factory=list)
    source: str = "none"
    multicast_supported: Optional[bool] = None

    @property
    def gpu_count(self) -> int:
        return len(self.gpus)

    def all_peers(self, indices: List[int]) -> bool:
        """True when every pair in ``indices`` can do P2P (NVSwitch: always)."""
        by = {g.index: g for g in self.gpus}
        for i in indices:
            for j in indices:
                if i != j and by[i].nvlink_peers and j not in by[i].nvlink_peers:
                    return False
        return True

    def to_dict(self) -> dict:
        return {"source": self.source, "multicast_supported": self.multicast_supported,
                "gpus": [g.__dict__ for g in self.gpus]}


def _numa_of_bus(bus_id: str) -> Optional[int]:
    """NVML / torch give "00000000:1B:00.0" or "0000:1b:00.0"; sysfs wants the 4-digit-domain lower-case form."""
    if not bus_id:
        return None
    parts = bus_id.lower().split(":")
    if len(parts) == 3:
        parts[0] = parts[0][-4:].rjust(4, "0")
    root = os.environ.get("B200MPI_SYSFS_ROOT", "")
    try:
        node = int(open(f"{root}/sys/bus/pci/devices/{':'.join(parts)}/numa_node").read().strip())
    except (OSError, ValueError):
        return None
    return node if node >= 0 else None


def _from_nvml() -> Optional[Topology]:
    try:
        import pynvml  # nvidia-ml-py
        pynvml.nvmlInit()
    except Exception:
        return None
    try:
        n = pynvml.nvmlDeviceGetCount()
        handles = [pynvml.nvmlDeviceGetHandleByIndex(i) for i in range(n)]
        gpus = []
        for i, h in enumerate(handles):
            name = pynvml.nvmlDeviceGetName(h)
            uuid = pynvml.nvmlDeviceGetUUID(h)
            mem = pynvml.nvmlDeviceGetMemoryInfo(h).total
            peers = []
            for j, hj in enumerate(handles):
                if i == j:
                    continue
                try:
                    st = pynvml.nvmlDeviceGetP2PStatus(h, hj, pynvml.NVML_P2P_CAPS_INDEX_NVLINK)
                    if st == pynvml.NVML_P2P_STATUS_OK:
                        peers.append(j)
                except Exception:
                    pass
            try:
                bus = pynvml.nvmlDeviceGetPciInfo(h).busId
                bus = bus if isinstance(bus, str) else bus.decode()
            except Exception:
                bus = ""
            gpus.append(GPU(i, uuid if isinstance(uuid, str) else uuid.decode(), name if isinstance(name, str) else name.decode(), int(mem), peers,
                            bus, _numa_of_bus(bus)))
        return Topology(gpus, "nvml")
    except Exception:
        return None
    finally:
        try:
            pynvml.nvmlShutdown()
        except Exception:
            pass


def _from_torch() -> Optional[Topology]:
    try:
        import torch
        if not torch.cuda.is_available():
            return None
        n = torch.cuda.device_count()
        gpus = []
        for i in range(n):
            p = torch.cuda.get_device_properties(i)
            peers = [j for j in range(n) if j != i and torch.cuda.can_device_access_peer(i, j)]
            try:
                bus = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
            except AttributeError:
                bus = ""
            gpus.append(GPU(i, str(getattr(p, "uuid", "")), p.name, int(p.total_memory), peers, bus, _numa_of_bus(bus)))
        return Topology(gpus, "torch")
    except Exception:
        return None


def discover_topology() -> Topology:
    fake = os.environ.get("B200MPI_FAKE_GPUS")
    if fake is not None:
        n = int(fake)
        nodes = int(os.environ.get("B200MPI_FAKE_NUMA_NODES", 0))     # e.g. 2: GPUs 0..n/2-1 on socket 0, the rest on socket 1 (HGX layout)
        return Topology([GPU(i, f"GPU-fake-{i}", "FakeB200", 180 << 30, [j for j in range(n) if j != i], f"0000:{0x1b + 0x10 * i:02x}:00.0",
                             (i * nodes // n) if nodes > 0 else None) for i in range(n)], "fake")
    vis = os.environ.get("CUDA_VISIBLE_DEVICES")
    topo = _from_nvml() or _from_torch() or Topology([], "none")
    if vis not in (None, "") and topo.source == "nvml":
        try:
            keep = [int(x) for x in vis.split(",") if x.strip() != ""]
            topo.gpus = [g for g in topo.gpus if g.index in keep]
        except ValueError:
            pass
    return topo
