"""Adasum reduction (the optional ``--use-adasum`` flag of the reference example,
examples/v2beta1/horovod/tensorflow_mnist.py:31-32,126-133; SURVEY.md §2.5 K6).

Adasum(a, b) = (1 - a.b / (2|a|^2)) a + (1 - a.b / (2|b|^2)) b, applied as a binary tree over the
ranks: orthogonal gradients add, parallel gradients average. Two device paths:

* ``B200MPI_ADASUM_KERNEL=1``: ``Communicator.adasum`` - ONE kernel per tensor (csrc/kernels/adasum.cu), each rank owns
  one slice of every vector, the tree levels run inside the launch over NVSwitch peer memory (S bytes pulled + S bytes
  pushed per rank, log2(N)+2 flag barriers). Power-of-two worlds, f32 / bf16 / f16, tensors up to
  ``Communicator.adasum_max_bytes``. Opt-in (tests/test_zzz_adasum_gpu.py is its numerics test).
* otherwise every rank gathers the N tensors (one b200mpi allgather kernel) and folds the tree locally in fp32 -
  identical bits on all ranks, O(N*S) scratch; fine for the example-scale models that use Adasum.
"""
from __future__ import annotations

import os
from typing import List

import torch


def _work(t: torch.Tensor) -> torch.Tensor:
    return t if t.dtype == torch.float64 else t.float()     # 16-bit floats are combined in fp32, doubles stay doubles


def adasum_pair(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    a32, b32 = _work(a), _work(b)
    dot = torch.dot(a32.flatten(), b32.flatten())
    na, nb = a32.pow(2).sum(), b32.pow(2).sum()
    ca = torch.where(na > 0, 1.0 - dot / (2.0 * na.clamp_min(1e-30)), torch.ones_like(dot))
    cb = torch.where(nb > 0, 1.0 - dot / (2.0 * nb.clamp_min(1e-30)), torch.ones_like(dot))
    return ca * a32 + cb * b32


def adasum_tree(tensors: List[torch.Tensor]) -> torch.Tensor:
    """Pairwise (recursive-halving order) fold; N need not be a power of two."""
    level = [_work(t) for t in tensors]
    while len(level) > 1:
        nxt = [adasum_pair(level[i], level[i + 1]) for i in range(0, len(level) - 1, 2)]
        if len(level) % 2:
            nxt.append(level[-1])
        level = nxt
    return level[0]


def _kernel_enabled() -> bool:
    return os.environ.get("B200MPI_ADASUM_KERNEL", "0") not in ("", "0", "false", "off")


def adasum_allreduce_(comm, tensor: torch.Tensor, stream=None) -> torch.Tensor:
    flat = tensor.contiguous().view(-1)
    if (_kernel_enabled() and not getattr(comm, "is_local", False) and hasattr(comm, "adasum_max_bytes")
            and 0 < flat.numel() * flat.element_size() <= comm.adasum_max_bytes(flat.dtype)):
        comm.adasum(flat, flat, stream=stream)
        if flat.data_ptr() != tensor.data_ptr():
            tensor.copy_(flat.view_as(tensor))
        return tensor
    work = flat if flat.dtype in (torch.float32, torch.bfloat16, torch.float16, torch.float64) else flat.float()   # the allgather kernel is byte-wise
    gathered = torch.empty(comm.world * work.numel(), dtype=work.dtype, device=work.device)
    comm.allgather(work, gathered, stream=stream)
    out = adasum_tree(list(gathered.view(comm.world, -1).unbind(0)))
    tensor.copy_(out.view_as(tensor).to(tensor.dtype))
    return tensor
