"""Data-parallel training engine over the b200mpi runtime.

The reference's only parallelism strategy is synchronous data parallelism by
delegation to Horovod (SURVEY.md §2.3: ``hvd.DistributedOptimizer`` averaging
gradients, ``BroadcastGlobalVariablesHook(0)``; examples/v2beta1/horovod/
tensorflow_mnist.py:133,143).  Horovod's engine = negotiate -> pack ready
tensors into a fusion buffer -> ncclAllReduce -> scale -> unpack -> optimizer.

GPU-first redesign:

* parameters and gradients live *inside symmetric windows* (peer-mapped, NVLS
  bound): autograd writes gradients straight into NVLink-visible memory, so
  there is no fusion-buffer pack/unpack copy at all;
* buckets are contiguous window regions in reverse-parameter order; when the
  last gradient of a bucket lands, ONE kernel on the comm stream does
  reduce-scatter + 1/N scale + weight-decay + momentum + parameter update +
  all-gather of the *updated parameters* (``b200mpi_allreduce_sgd_sym``) —
  no separate scale kernel, no optimizer kernel, momentum sharded 1/N;
* the whole step (forward, backward, hooks, comm kernels) is captured once in
  a CUDA graph and replayed: no per-step launch overhead, no tracing compiler.
"""
from __future__ import annotations

import contextlib
import os
from dataclasses import dataclass, field
from typing import Callable, List, Optional

import torch
import torch.nn as nn

from ..ops import fused_bn
from ..runtime.comm import Communicator, Window
from ..utils import fault, nvtx
from .lr_schedule import LRSchedule


def _align(n: int, a: int) -> int:
    return (n + a - 1) // a * a


MAX_PARAM_GROUPS = 256   # the fused kernel's group map holds one byte per vector
MAX_LARS_BUCKET_PARAMS = 1024   # the fused LARS kernels keep one trust ratio per parameter of a bucket in shared memory
LARS_EPS = 1e-8                 # the fixed epsilon of the trust ratio's denominator (the kernels' kLarsEps)
_GROUP_KEYS = {"params", "lr", "momentum", "weight_decay", "nesterov", "lars"}


def _resolve_param_groups(model: nn.Module, param_groups: Optional[list], lr: float, momentum: float, weight_decay: float,
                          nesterov: bool, lars: bool = False):
    """torch-style ``param_groups`` -> (members, values, lars flags): group 0 holds the trainable parameters no group lists,
    with the trainer-level values; group k >= 1 is ``param_groups[k - 1]``, its missing keys taken from the trainer."""
    trainable = [p for p in model.parameters() if p.requires_grad]
    groups = list(param_groups or [])
    if len(groups) + 1 > MAX_PARAM_GROUPS:
        raise ValueError(f"{len(groups)} parameter groups: at most {MAX_PARAM_GROUPS - 1} besides the implicit group 0")
    known = {id(p) for p in trainable}
    taken = set()
    members, values, lars_flags = [], [[lr, momentum, weight_decay]], [bool(lars)]
    for k, g in enumerate(groups):
        if not isinstance(g, dict) or "params" not in g:
            raise ValueError(f"parameter group {k}: expected a dict with a 'params' entry")
        unknown = set(g) - _GROUP_KEYS
        if unknown:
            raise ValueError(f"parameter group {k}: unsupported keys {sorted(unknown)} (lr, momentum, weight_decay, lars)")
        if "lars" in g and not isinstance(g["lars"], bool):
            raise ValueError(f"parameter group {k}: 'lars' must be a bool, got {g['lars']!r}")
        if "nesterov" in g and bool(g["nesterov"]) != bool(nesterov):
            raise ValueError(f"parameter group {k}: nesterov is a trainer-wide setting ({nesterov}), not per group")
        ps = [g["params"]] if isinstance(g["params"], torch.Tensor) else list(g["params"])
        for p in ps:
            if id(p) not in known:
                raise ValueError(f"parameter group {k}: a tensor of shape {tuple(p.shape)} is not a trainable parameter of the model")
            if id(p) in taken:
                raise ValueError(f"parameter group {k}: a parameter of shape {tuple(p.shape)} is listed twice")
            taken.add(id(p))
        members.append(ps)
        values.append([float(g.get("lr", lr)), float(g.get("momentum", momentum)), float(g.get("weight_decay", weight_decay))])
        lars_flags.append(g.get("lars", bool(lars)))
    members.insert(0, [p for p in trainable if id(p) not in taken])
    return members, values, lars_flags


@dataclass
class Bucket:
    index: int
    start: int            # element offset in the flat buffers
    numel: int            # padded to a multiple of 8 elements (16-byte vectors for fp32 and bf16)
    params: List[nn.Parameter] = field(default_factory=list)
    pending: int = 0
    momentum: Optional[torch.Tensor] = None  # this rank's shard
    lars: bool = False                       # holds a LARS parameter: runs the fused LARS kernels
    param_table: Optional[torch.Tensor] = None   # [len(params), 2] uint8 {group, lars}, bucket-local parameter order
    trust: Optional[torch.Tensor] = None     # LARS buckets: trust ratio of each parameter at the last synchronising step
    ema: Optional[torch.Tensor] = None       # ema_decay: this rank's shard of the weight average, sharded like momentum


class FlatModelState:
    """Re-homes a module's parameters and gradients into two symmetric windows
    with identical element layout (fp32), bucketed in reverse registration order
    (the order backward produces them).

    ``bf16_params=True`` adds a third window with the same element layout in bf16: matrix-shaped
    parameters (conv / linear weights) become bf16 leaves that view it, their fp32 masters stay in
    the parameter window and the fused SGD kernel refreshes the shadow in the same pass
    (``lowp_win``). Forward then needs no per-layer fp32->bf16 weight cast and backward no
    bf16->fp32 gradient cast + accumulate: ~3 small kernels per layer disappear from the step."""

    def __init__(self, module: nn.Module, comm: Communicator, bucket_bytes: int = 32 << 20, bf16_params: bool = False,
                 group_of: Optional[dict] = None, lars_of: Optional[dict] = None):
        """``group_of`` (parameter -> group index, missing: 0) builds ``group_map``: one uint8 group id per 4-element
        vector of the flat buffers, which the grouped fused SGD kernel reads per vector. ``lars_of`` (parameter -> bool,
        missing: False) builds ``param_map`` and each bucket's ``{group, lars}`` parameter table for the fused LARS
        kernels."""
        self.comm = comm
        self.bf16_params = bf16_params
        params = [p for p in module.parameters() if p.requires_grad]
        if any(p.dtype != torch.float32 for p in params):
            raise ValueError("FlatModelState expects fp32 master parameters (use autocast for bf16 compute)")
        self.params = params
        order = list(reversed(params))
        self.buckets: List[Bucket] = []
        self.param_slot = {}
        off = 0
        cur = Bucket(0, 0, 0)
        cap = max(bucket_bytes // 4, 1)
        # The LAST bucket (the earliest layers) is the one whose allreduce+SGD cannot hide behind backward. With
        # B200MPI_TAIL_BUCKET_BYTES=<n> (e.g. 4194304) it is capped at n bytes so the exposed tail of the step is one short
        # kernel. With world > 1 opt-in (0 = off): it was on during round 2's 8-GPU session, whose bench record was lost; bench.py
        # measures it as its second multi-GPU candidate.
        # Single-GPU default: 4 MiB (there the last bucket's kernel is exposed in full - it can only start when backward has
        # finished - and nothing else changes: same kernel, one more launch).
        tail_cap = int(os.environ.get("B200MPI_TAIL_BUCKET_BYTES", (4 << 20) if (comm.world == 1 and comm.device != "cpu") else 0)) // 4
        pad = 64 if bf16_params else 4
        remaining = sum(_align(p.numel(), pad) for p in order)
        tail_started = False
        for p in order:
            # keep every tensor 16-byte aligned; with a bf16 shadow, 64 elements so the bf16 views handed to
            # cuDNN start on 128-byte boundaries as well
            n = _align(p.numel(), pad)
            start_tail = bool((not tail_started) and len(cur.params) > 0 and remaining <= tail_cap and remaining < cap)
            tail_started = tail_started or start_tail
            remaining -= n
            if cur.params and (cur.numel + n > cap or start_tail):
                cur.numel = _align(cur.numel, 8)
                off = cur.start + cur.numel
                self.buckets.append(cur)
                cur = Bucket(len(self.buckets), off, 0)
            self.param_slot[p] = (cur.index, cur.start + cur.numel)
            cur.params.append(p)
            cur.numel += n
        cur.numel = _align(cur.numel, 8)
        self.buckets.append(cur)
        self.total = cur.start + cur.numel
        self.param_win: Window = comm.alloc_window(self.total * 4)
        self.grad_win: Window = comm.alloc_window(self.total * 4)
        self.flat_param = self.param_win.tensor(torch.float32, numel=self.total)
        self.flat_grad = self.grad_win.tensor(torch.float32, numel=self.total)
        self.flat_param.zero_()
        self.flat_grad.zero_()
        self.lowp_win: Optional[Window] = None
        self.flat_lowp = None
        self.lowp_params = set()
        self.grad_view = {}
        if bf16_params:
            self.lowp_win = comm.alloc_window(self.total * 2)
            self.flat_lowp = self.lowp_win.tensor(torch.bfloat16, numel=self.total)
            self.flat_lowp.zero_()
        for p in params:
            _, start = self.param_slot[p]
            n = p.numel()
            pv = self.flat_param[start:start + n].as_strided(p.size(), p.stride())
            pv.copy_(p.data)
            gv = self.flat_grad[start:start + n].as_strided(p.size(), p.stride())
            self.grad_view[p] = gv
            if bf16_params and p.dim() >= 2:
                lv = self.flat_lowp[start:start + n].as_strided(p.size(), p.stride())
                lv.copy_(pv)
                p.data = lv      # bf16 leaf; master = flat_param slot; gradient arrives in bf16 and is
                p.grad = None    # gathered into the fp32 window per bucket (DataParallelTrainer._gather_grads)
                self.lowp_params.add(p)
            else:
                p.data = pv
                p.grad = gv
        for b in self.buckets:
            b.momentum = torch.zeros(comm.slice_elems(b.numel, torch.float32), device=self.flat_param.device)
        self.group_map: Optional[torch.Tensor] = None
        if group_of is not None:
            # every slot starts on a vector and is padded to whole vectors, so each vector lies in one parameter; its padding
            # takes that parameter's group, the bucket tails (zeros in every buffer) group 0
            gmap = torch.zeros(self.total // 4, dtype=torch.uint8)
            for p in params:
                start = self.param_slot[p][1]
                gmap[start // 4:(start + _align(p.numel(), pad)) // 4] = group_of.get(p, 0)
            self.group_map = gmap.to(self.flat_param.device)
        self.param_map: Optional[torch.Tensor] = None
        if lars_of is not None:
            # bucket-local parameter index of each vector: a parameter's padding takes its index, the bucket tail the index
            # one past the bucket's last parameter (the kernels' trust-1 dummy entry)
            pmap = torch.zeros(self.total // 4, dtype=torch.int32)
            for b in self.buckets:
                pmap[b.start // 4:(b.start + b.numel) // 4] = len(b.params)
                for k, p in enumerate(b.params):
                    start = self.param_slot[p][1]
                    pmap[start // 4:(start + _align(p.numel(), pad)) // 4] = k
            self.param_map = pmap.to(torch.uint16).to(self.flat_param.device)
            group_of = group_of or {}
            for b in self.buckets:
                b.lars = any(lars_of.get(p, False) for p in b.params)
                if b.lars and len(b.params) > MAX_LARS_BUCKET_PARAMS:
                    raise ValueError(f"bucket {b.index} holds {len(b.params)} parameters; the fused LARS kernels take at "
                                     f"most {MAX_LARS_BUCKET_PARAMS} per bucket: use a smaller bucket_bytes")
                b.param_table = torch.tensor([[group_of.get(p, 0), int(bool(lars_of.get(p, False)))] for p in b.params],
                                             dtype=torch.uint8).to(self.flat_param.device)
                if b.lars:
                    b.trust = torch.ones(len(b.params), dtype=torch.float32, device=self.flat_param.device)

    def bucket_param_map(self, b: Bucket) -> torch.Tensor:
        """The slice of ``param_map`` covering bucket ``b``."""
        return self.param_map[b.start // 4:(b.start + b.numel) // 4]

    def bucket_group_map(self, b: Bucket) -> torch.Tensor:
        """The slice of ``group_map`` covering bucket ``b`` (``b.start`` and ``b.numel`` are multiples of 8 elements)."""
        return self.group_map[b.start // 4:(b.start + b.numel) // 4]

    def broadcast_parameters(self, root: int = 0) -> None:
        """K3: rank-0 state to everyone (tensorflow_mnist.py:143)."""
        if self.comm.world > 1:
            mode = os.environ.get("B200MPI_PARAM_BROADCAST", "window")
            if mode == "window" and hasattr(self.comm, "broadcast_window"):   # zero-copy: the parameters already live in a symmetric window
                self.comm.broadcast_window(self.param_win, 0, self.total * 4, root=root)
            elif mode == "staged" and hasattr(self.comm, "set_pipe"):
                # the barrier-based staged kernel, exactly what round 1 ran on 8 GPUs (bench.py's conservative configuration)
                self.comm.set_pipe(min_bytes=1 << 62)
                self.comm.set_reg(0)
                try:
                    self.comm.broadcast(self.flat_param, root=root)
                finally:
                    self.comm.set_pipe(min_bytes=8 << 20)
                    self.comm.set_reg(1)
            else:
                self.comm.broadcast(self.flat_param, root=root)
        self.refresh_lowp()

    def refresh_lowp(self) -> None:
        """Re-derive the bf16 shadow from the fp32 masters (after a broadcast, a checkpoint load or an
        optimizer that does not write it itself)."""
        if self.flat_lowp is not None:
            self.flat_lowp.copy_(self.flat_param)

    def master_state(self) -> dict:
        """fp32 master copy of every re-homed parameter, keyed by its index in ``module.parameters()`` order —
        what a checkpoint should store when ``bf16_params`` is on (the module itself holds bf16 leaves)."""
        out = {}
        for i, p in enumerate(self.params):
            start = self.param_slot[p][1]
            out[i] = self.flat_param[start:start + p.numel()].as_strided(p.size(), p.stride())
        return out

    def zero_grad(self) -> None:
        self.flat_grad.zero_()


class DataParallelTrainer:
    """User-facing training loop object.

    >>> trainer = DataParallelTrainer(model, loss_fn, comm, lr=0.1, momentum=0.9)
    >>> loss = trainer.step(images_pinned_cpu, labels_pinned_cpu)   # returns a device scalar

    ``step`` performs, every call: H2D copy of the batch (from the caller's
    pinned host tensors), forward + backward under bf16 autocast, bucketed fused
    allreduce+SGD on the comm stream overlapped with backward, and leaves the
    loss on the device (``float(loss)`` is the D2H read).

    ``param_groups`` takes ``torch.optim.SGD``-style groups, e.g. no weight decay on BatchNorm and biases::

        no_wd = [p for n, p in model.named_parameters() if p.dim() == 1]
        trainer = DataParallelTrainer(model, loss_fn, comm, lr=0.1, weight_decay=5e-5,
                                      param_groups=[{"params": no_wd, "weight_decay": 0.0}])

    Each group may set ``lr``, ``momentum`` and ``weight_decay``; missing keys take the trainer-level values. Trainable
    parameters in no group form group 0 with the trainer-level values, so the groups given are 1, 2, ... in
    ``trainer.param_groups`` and ``set_lr(lr, group=k)``. All three optimizer paths (fused kernel, ``fused_optimizer=False``,
    ``comm_backend="nccl"``) apply the same per-group update.

    ``lars=True`` turns on LARS (You et al., 2017) for group 0 and is the default of groups without a ``"lars"`` key; the
    MLPerf ResNet recipe leaves BatchNorm and biases out of it and out of weight decay::

        no_lars = [p for p in model.parameters() if p.dim() == 1]
        trainer = DataParallelTrainer(model, loss_fn, comm, lr=..., momentum=0.9, weight_decay=5e-5,
                                      lars=True, trust_coefficient=0.001,
                                      param_groups=[{"params": no_lars, "weight_decay": 0.0, "lars": False}])

    At each synchronising step every parameter tensor ``w`` of a LARS group, with ``g`` its world-averaged gradient and both
    norms taken over the fp32 master before the update, gets ``trust = eta * |w| / (|g| + wd * |w| + 1e-8)`` (``trust = 1``
    when ``|w|`` or ``|g|`` is 0), ``d = trust * (g + wd * w)``, ``m = mu * m + d`` and ``w -= lr * (d + mu * m if nesterov
    else m)``; other parameters keep the plain update (``trust = 1``). ``eta`` is ``trust_coefficient``, trainer-wide and
    fixed at construction. Apex's ``LARC(clip=False)`` differs only where a norm is 0: it then also drops the weight decay.
    ``lars_trust_ratios()`` returns the trust ratios of the last synchronising step.

    ``ema_decay=d`` (``0 < d < 1``) keeps an exponential moving average of the fp32 master of every trainable parameter, as
    tf_cnn_benchmarks' ``--moving_average_decay`` does with ``tf.train.ExponentialMovingAverage(d, num_updates=step)``. It
    starts at the broadcast parameters; the k-th synchronising step (k = 1, 2, ..., every step that updated the parameters,
    the CUDA-graph capture's warm-up steps included) applies ``e = e + c_k * (p - e)`` to the updated parameters ``p`` with
    ``c_k = 1 - min(d, (1 + k) / (10 + k))``. The fused kernels do it in the same pass as the update, on the slice each rank
    owns. BatchNorm running statistics are not averaged: they already are averages, and an evaluation under the averaged
    weights uses the live ones::

        trainer = DataParallelTrainer(model, loss_fn, comm, lr=0.1, ema_decay=0.9999)
        ...
        with trainer.ema_weights():            # collective when world > 1
            print(trainer.evaluate(x, y))

    ``lr_schedule=LRSchedule...`` (``mpi_operator_b200.parallel.lr_schedule``) makes each group's learning rate
    ``fp32(base * m(k))``, ``base`` the group's ``lr`` and ``k`` the number of synchronising steps before this one (the
    CUDA-graph capture's warm-up steps included, ``no_sync()`` steps not). One single-CTA kernel on the compute stream
    writes the rates into the device tables before each synchronising backward, so captured replays follow the schedule.
    ``set_lr`` then sets the base rate, ``param_groups`` and checkpoints report base rates and ``current_lrs()`` the rates
    of the last step. MLPerf's LARS recipe, linear warm-up then quadratic decay::

        sched = LRSchedule.polynomial(total_steps=steps, power=2, warmup_steps=warmup)
        trainer = DataParallelTrainer(model, loss_fn, comm, lr=peak_lr, lars=True, lr_schedule=sched, ...)
    """

    def __init__(self, model: nn.Module, loss_fn: Callable, comm: Communicator, *, lr: float, momentum: float = 0.9,
                 weight_decay: float = 0.0, nesterov: bool = False, bucket_bytes: Optional[int] = None,
                 autocast_dtype: Optional[torch.dtype] = torch.bfloat16, channels_last: bool = True,
                 cuda_graph: bool = True, fused_optimizer: bool = True, algo: Optional[str] = None,
                 comm_backend: str = "b200mpi", bf16_params: Optional[bool] = None, async_h2d: Optional[bool] = None,
                 param_groups: Optional[list] = None, lars: bool = False, trust_coefficient: float = 0.001,
                 ema_decay: Optional[float] = None, lr_schedule: Optional[LRSchedule] = None):
        if lr_schedule is not None and not isinstance(lr_schedule, LRSchedule):
            raise ValueError(f"lr_schedule must be None or an LRSchedule, got {lr_schedule!r}")
        if ema_decay is not None and not (isinstance(ema_decay, (int, float)) and not isinstance(ema_decay, bool)
                                          and 0.0 < float(ema_decay) < 1.0):
            raise ValueError(f"ema_decay must be None or a number in (0, 1), got {ema_decay!r}")
        if not isinstance(lars, bool):
            raise ValueError(f"lars must be a bool, got {lars!r}")
        if not (isinstance(trust_coefficient, (int, float)) and float(trust_coefficient) > 0
                and float(trust_coefficient) != float("inf")):
            raise ValueError(f"trust_coefficient must be a finite number > 0, got {trust_coefficient!r}")
        self.trust_coefficient = float(trust_coefficient)
        self.comm = comm
        self.device = torch.device("cuda", comm.device) if comm.device != "cpu" else torch.device("cpu")
        self._cuda = self.device.type == "cuda"
        if bf16_params is None:
            # Default on for single-GPU CUDA runs (it removes the per-layer weight casts). With world > 1 the fused kernel pushes the bf16 shadow to every peer with unicast 8-byte stores
            # (no multimem form yet) and that path has not been measured on more than one GPU: opt-in there
            # (B200MPI_BF16_PARAMS=1). The CPU debug path keeps fp32 leaves unless asked.
            bf16_params = os.environ.get("B200MPI_BF16_PARAMS", "1" if (self._cuda and comm.world == 1) else "0") == "1"
        self.bf16_params = bool(bf16_params) and autocast_dtype == torch.bfloat16
        self.loss_fn = loss_fn
        self.autocast_dtype = autocast_dtype
        self.channels_last = channels_last
        self.use_graph = cuda_graph
        self.fused = fused_optimizer and comm_backend == "b200mpi"
        self.algo = algo
        self.backend = comm_backend  # "b200mpi" | "nccl" (baseline: stock NCCL via torch.distributed)
        self.nesterov = nesterov
        model = model.to(self.device)
        if channels_last:
            model = model.to(memory_format=torch.channels_last)
        self.model = model
        bucket_bytes = bucket_bytes or int(os.environ.get("B200MPI_BUCKET_BYTES", 32 << 20))
        names = {p: n for n, p in model.named_parameters()}
        self._has_groups = param_groups is not None
        members, values, lars_flags = _resolve_param_groups(model, param_groups, lr, momentum, weight_decay, nesterov, lars)
        self._group_names = [[names[p] for p in ps] for ps in members]
        self._group_vals = values        # host copy of group_hyper, [[lr, momentum, weight_decay], ...]
        self._group_lars = lars_flags    # per group: LARS on or off
        # LARS reads {lr, momentum, weight_decay} from the group table even without param_groups (one row)
        self._lars = any(lars_flags)
        self._tabled = self._has_groups or self._lars
        group_of = {p: k for k, ps in enumerate(members) for p in ps} if self._tabled else None
        lars_of = {p: lars_flags[k] for k, ps in enumerate(members) for p in ps} if self._lars else None
        self.state = FlatModelState(model, comm, bucket_bytes, bf16_params=self.bf16_params, group_of=group_of,
                                    lars_of=lars_of)
        self.state.broadcast_parameters(0)
        # {lr, momentum, weight_decay} on the device: graph replays follow schedules
        self.hyper = torch.tensor([lr, momentum, weight_decay], device=self.device, dtype=torch.float32)
        comm.set_hyper(self.hyper)
        self._lr, self._mu, self._wd = lr, momentum, weight_decay
        # with param_groups: one {lr, momentum, weight_decay} row per group on the device, read by the kernels the same way
        self.group_hyper = torch.tensor(values, device=self.device, dtype=torch.float32) if self._tabled else None
        # learning-rate schedule: the table, each group's base rate (float64) and the step count k on the device; the
        # kernel rewrites the lr column of hyper / group_hyper from them every synchronising step
        self.lr_schedule = lr_schedule
        if lr_schedule is not None:
            self._lr_table = torch.tensor(lr_schedule.table(), dtype=torch.float64, device=self.device)
            self._lr_base = torch.tensor([float(v[0]) for v in values], dtype=torch.float64, device=self.device)
            self._lr_step = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._lars_board = self._lars_scratch = None
        if self._lars:
            self._alloc_lars()
        # weight average: {d as fp32 widened, updates so far} on the device, read by the fused kernels (graph replays follow
        # it); the fused path keeps one shard per bucket beside the momentum, the unfused paths one full flat copy
        self.ema_decay = None if ema_decay is None else float(torch.tensor(float(ema_decay), dtype=torch.float32))
        self._ema_sched = None
        self._flat_ema = None
        self._in_ema = False
        if self.ema_decay is not None:
            self._ema_sched = torch.tensor([self.ema_decay, 0.0], dtype=torch.float64, device=self.device)
            if self.fused:
                for b in self.state.buckets:
                    b.ema = torch.zeros_like(b.momentum)
            self._set_ema(self.state.flat_param)
        self.comm_stream = torch.cuda.Stream(device=self.device, priority=-1) if self._cuda else None
        self._graph: Optional[torch.cuda.CUDAGraph] = None
        self._static_x = self._static_y = None
        self._loss = torch.zeros((), device=self.device)
        self._launches_per_step = 0
        self._sync = True
        self._carry = False
        # B200MPI_ASYNC_H2D=1: inputs go host -> staging buffer on a copy stream (overlapping the previous step's compute),
        # then device -> device into the graph's static input, so the copy overlaps compute. Default on.
        self.async_h2d = os.environ.get("B200MPI_ASYNC_H2D", "1") == "1" if async_h2d is None else bool(async_h2d)
        self._copy_stream = torch.cuda.Stream(device=self.device) if (self.async_h2d and self._cuda) else None
        self._stage_x = self._stage_y = None
        self._pending_batch = None
        # the 104 `num_batches_tracked += 1` kernels of a ResNet-101 step become one multi-tensor add;
        # B200MPI_DEFER_NBT=0 restores one add per BN layer
        self._defer_nbt = os.environ.get("B200MPI_DEFER_NBT", "1" if self._cuda else "0") == "1"
        self._graph_ops: list = []   # collectives recorded in the CUDA graph: replays launch them without the host
        self._replays = 0
        if hasattr(comm, "add_stat_source"):
            comm.add_stat_source(self._replayed_ops)
        self._folded_ops: list = []  # totals of graphs that were since re-captured
        self._fault = fault.injector(comm.rank)  # $B200MPI_FAULT recovery tests; disarmed when unset
        self._eval_graphs: dict = {}    # evaluate() under cuda_graph: input shape -> (graph, static x, static y, stats, top-k)
        hooks = {}
        for b in self.state.buckets:
            for p in b.params:
                hooks[p] = self._make_hook(b)
                p.register_post_accumulate_grad_hook(hooks[p])
        # fused BN layers write dgamma/dbeta directly into the flat gradient views and report readiness
        # themselves (mpi_operator_b200.ops.fused_bn): no AccumulateGrad add kernels for 2 x #BN params
        for mod in model.modules():
            if isinstance(mod, nn.BatchNorm2d) and mod.affine and mod.weight in hooks:
                ready = (lambda param, _h=hooks: _h[param](param))
                ready.accumulating = lambda: (not self._sync) or self._carry
                mod._b200_grad_ready = ready
        if self.backend == "nccl":
            import torch.distributed as dist
            self._dist = dist
        if self._cuda:
            torch.cuda.synchronize(self.device)
        if comm.world > 1:
            comm.host_barrier()

    # ---------------------------------------------------------- hyper --
    def set_lr(self, lr: float, group: Optional[int] = None) -> None:
        """Learning rate of every group (``group=None``) or of group ``group`` (an index into ``param_groups``; group 0
        holds the trainer-level values). Takes effect from the next step, CUDA-graph replays included. With ``lr_schedule``
        it sets the base rate the schedule multiplies."""
        if group is not None and not 0 <= group < len(self._group_vals):
            raise IndexError(f"group {group} out of range: the trainer has {len(self._group_vals)} parameter groups")
        if self.lr_schedule is not None:
            if group is None or group == 0:
                self._lr = lr
            for k in (range(len(self._group_vals)) if group is None else (group,)):
                self._group_vals[k][0] = lr
                self._lr_base[k] = float(lr)
            return
        if group is None or group == 0:
            self._lr = lr
            self.hyper[0] = lr
        for k in (range(len(self._group_vals)) if group is None else (group,)):
            self._group_vals[k][0] = lr
        if self.group_hyper is not None:
            if group is None:
                self.group_hyper[:, 0] = lr
            else:
                self.group_hyper[group, 0] = lr

    def _schedule_step(self) -> None:
        """Write the scheduled rates of step k into the lr column of the tables and advance k."""
        sch = self.lr_schedule
        if self._cuda:
            self.comm.lr_schedule(self._lr_table, sch.form, len(sch.boundaries), self._lr_step, self._lr_base, self.hyper,
                                  self.group_hyper, stream=torch.cuda.current_stream(self.device))
            return
        k = int(self._lr_step)
        self._write_rates(k)
        self._lr_step += 1

    def _write_rates(self, k: int) -> None:
        """The rates of step ``k`` (``LRSchedule.rate``: the kernel's bits) into the lr column of the tables."""
        rates = [self.lr_schedule.rate(v[0], k) for v in self._group_vals]
        self.hyper[0] = rates[0]
        if self.group_hyper is not None:
            self.group_hyper[:, 0] = torch.tensor(rates, dtype=torch.float32)

    def current_lrs(self) -> list:
        """Each group's learning rate as the last synchronising step used it (with a schedule: the base rates before the
        first step). Reading it synchronises with the device."""
        if self.group_hyper is not None:
            return [float(v) for v in self.group_hyper[:, 0].tolist()]
        return [float(self.hyper[0])]

    @property
    def lr_schedule_step(self) -> int:
        """k: the synchronising steps the schedule has seen (reading it synchronises with the device)."""
        return int(self._lr_step) if self.lr_schedule is not None else 0

    @property
    def param_groups(self) -> list:
        """``[{"params": [parameter names], "lr": ..., "momentum": ..., "weight_decay": ..., "lars": ...}, ...]``, group 0
        (parameters in no given group, trainer-level values) first. A copy: change values with ``set_lr``."""
        return [{"params": list(n), "lr": v[0], "momentum": v[1], "weight_decay": v[2], "lars": f}
                for n, v, f in zip(self._group_names, self._group_vals, self._group_lars)]

    def _alloc_lars(self) -> None:
        """Norm board (a symmetric window of [P][world] float pairs) and per-rank scratch of the fused LARS kernels, sized
        for the largest LARS bucket; one of each serves every bucket, as the buckets run in stream order."""
        st = self.state
        lb = [b for b in st.buckets if b.lars]
        if not (self.fused and lb) or self._lars_board is not None:
            return
        P = max(len(b.params) for b in lb)
        self._lars_board = self.comm.alloc_window(_align(P * self.comm.world * 8, 16))
        nbytes = max(self.comm.lars_scratch_bytes(b.numel, len(b.params)) for b in lb)
        self._lars_scratch = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)

    def lars_trust_ratios(self) -> dict:
        """``{parameter name: trust ratio}`` of every LARS parameter at the last synchronising step (1.0 before the first).
        Reading it synchronises with the device."""
        names = {p: n for n, p in self.model.named_parameters()}
        out = {}
        for b in self.state.buckets:
            if b.lars:
                vals, flags = b.trust.tolist(), b.param_table[:, 1].tolist()
                out.update({names[p]: v for p, v, f in zip(b.params, vals, flags) if f})
        return out

    @property
    def launches_per_step(self) -> int:
        return self._launches_per_step

    def _replayed_ops(self) -> list:
        out = {(o["op"], o["algo"]): dict(o) for o in self._folded_ops}
        for o in self._graph_ops:
            m = out.setdefault((o["op"], o["algo"]), {"op": o["op"], "algo": o["algo"], "calls": 0, "bytes": 0})
            m["calls"] += o["calls"] * self._replays
            m["bytes"] += o["bytes"] * self._replays
        return list(out.values())

    # ---------------------------------------------------------- hooks --
    def _make_hook(self, bucket: Bucket):
        def hook(_param):
            if not self._sync:
                return
            bucket.pending -= 1
            if bucket.pending == 0:
                self._reduce_bucket(bucket)
        return hook

    def _gather_grads(self, b: Bucket) -> None:
        """bf16_params mode: autograd left each matrix parameter's gradient in a bf16 tensor of its own
        (``p.grad`` was None, so AccumulateGrad stole the buffer instead of adding); one multi-tensor
        copy per bucket casts them into the fp32 gradient window. Parameters that got no gradient keep
        the zeros written by ``zero_grad``."""
        st = self.state
        dst, src = [], []
        for p in b.params:
            if p in st.lowp_params and p.grad is not None:
                dst.append(st.grad_view[p])
                src.append(p.grad)
        if dst:
            torch._foreach_copy_(dst, src)
        for p in b.params:
            if p in st.lowp_params:
                p.grad = None

    def _reduce_bucket(self, b: Bucket) -> None:
        st = self.state
        if st.lowp_params:
            self._gather_grads(b)
        if not self._cuda:  # CPU debug path (tests/test_trainer_cpu.py): same bucket logic, no streams
            self._reduce_bucket_body(b)
            b.pending = -1
            return
        main = torch.cuda.current_stream(self.device)
        ev = torch.cuda.Event()
        ev.record(main)
        self.comm_stream.wait_event(ev)
        with torch.cuda.stream(self.comm_stream), nvtx.range(f"b200mpi.bucket@{b.start}"):
            self._reduce_bucket_body(b)
        b.pending = -1  # fired

    def _reduce_bucket_body(self, b: Bucket) -> None:
        st = self.state
        ema = {"ema": b.ema, "ema_sched": self._ema_sched} if b.ema is not None else {}
        if self.backend == "nccl":
            g = st.flat_grad[b.start:b.start + b.numel]
            if self.comm.world > 1:
                self._dist.all_reduce(g, op=self._dist.ReduceOp.AVG)
        elif self.fused and b.lars:
            self.comm.allreduce_lars_window(st.grad_win, b.start * 4, st.param_win, b.start * 4, b.momentum, b.numel,
                                            torch.float32, group_hyper=self.group_hyper,
                                            param_map=st.bucket_param_map(b), param_table=b.param_table,
                                            board_win=self._lars_board, board_off=0, scratch=self._lars_scratch,
                                            trust_coefficient=self.trust_coefficient, nesterov=self.nesterov,
                                            lowp_win=st.lowp_win, lowp_off=b.start * 2, algo=self.algo,
                                            stream=self.comm_stream, trust_out=b.trust, **ema)
        elif self.fused and self._has_groups:
            self.comm.allreduce_sgd_window(st.grad_win, b.start * 4, st.param_win, b.start * 4, b.momentum,
                                           b.numel, torch.float32, lr=self._lr, momentum_coef=self._mu,
                                           weight_decay=self._wd, nesterov=self.nesterov,
                                           lowp_win=st.lowp_win, lowp_off=b.start * 2, algo=self.algo,
                                           stream=self.comm_stream, group_map=st.bucket_group_map(b),
                                           group_hyper=self.group_hyper, **ema)
        elif self.fused:
            self.comm.allreduce_sgd_window(st.grad_win, b.start * 4, st.param_win, b.start * 4, b.momentum,
                                           b.numel, torch.float32, lr=self._lr, momentum_coef=self._mu,
                                           weight_decay=self._wd, nesterov=self.nesterov,
                                           lowp_win=st.lowp_win, lowp_off=b.start * 2, algo=self.algo,
                                           stream=self.comm_stream, **ema)
        else:
            self.comm.allreduce_window(st.grad_win, b.start * 4, b.numel, torch.float32, op="avg",
                                       algo=self.algo, stream=self.comm_stream)

    def _unfused_sgd(self) -> None:
        """Plain flat SGD (used by the NCCL baseline and fused_optimizer=False)."""
        st = self.state
        if not hasattr(self, "_flat_mom"):
            self._flat_mom = torch.zeros_like(st.flat_param)
        if self._tabled:
            # the fused kernel's per-vector update: each 4-element vector takes its group's row of the table
            if not hasattr(self, "_group_index"):
                self._group_index = st.group_map.long()
            h = self.group_hyper[self._group_index]
            lr, mu, wd = h[:, 0:1], h[:, 1:2], h[:, 2:3]
            p, m = st.flat_param.view(-1, 4), self._flat_mom.view(-1, 4)
            g = st.flat_grad.view(-1, 4) + wd * p
            if self._lars:
                g = g * self._unfused_trust()
            m.mul_(mu).add_(g)
            p.sub_(lr * (g + mu * m if self.nesterov else m))
            st.refresh_lowp()
            return
        g = st.flat_grad
        if self._wd:
            g = g.add(st.flat_param, alpha=self._wd)
        self._flat_mom.mul_(self.hyper[1]).add_(g)
        upd = g.add(self._flat_mom, alpha=self._mu) if self.nesterov else self._flat_mom
        st.flat_param.sub_(upd * self.hyper[0])
        st.refresh_lowp()

    def _unfused_ema(self) -> None:
        """The fused kernels' weight average on the full flat buffers (NCCL baseline and fused_optimizer=False); within 1 ulp
        of the fused result, which rounds the product and the sum once."""
        d, k = self._ema_sched[0], self._ema_sched[1]
        c = (1.0 - torch.minimum(d, (1.0 + k) / (10.0 + k))).float()
        self._flat_ema.addcmul_(self.state.flat_param - self._flat_ema, c)

    def _unfused_trust(self) -> torch.Tensor:
        """LARS trust ratio of every 4-element vector of the flat buffers ([total / 4, 1]; 1 outside LARS parameters), from
        the averaged gradients and the masters before the update; also stored as each bucket's ``trust``."""
        st = self.state
        if not hasattr(self, "_lars_index"):
            # vector -> row of the parameter list below; bucket tails the trailing row, which holds trust 1
            lp = [p for b in st.buckets for p in b.params]
            self._lars_params = lp
            self._lars_rows = {p: k for k, p in enumerate(lp)}
            idx = torch.full((st.total // 4,), len(lp), dtype=torch.long)
            pmap = st.param_map.cpu().long()
            for b in st.buckets:
                sl = slice(b.start // 4, (b.start + b.numel) // 4)
                first = self._lars_rows[b.params[0]]
                local = pmap[sl]
                idx[sl] = torch.where(local < len(b.params), local + first, torch.full_like(local, len(lp)))
            self._lars_index = idx.to(st.flat_param.device)
            self._lars_flag = torch.tensor([bool(b.param_table[k, 1]) for b in st.buckets for k in range(len(b.params))],
                                           device=st.flat_param.device)
            self._lars_group = torch.tensor([int(b.param_table[k, 0]) for b in st.buckets for k in range(len(b.params))],
                                            device=st.flat_param.device, dtype=torch.long)
        lp = self._lars_params
        views = [(st.param_slot[p][1], p.numel()) for p in lp]
        wn = torch.stack(torch._foreach_norm([st.flat_param[s:s + n] for s, n in views]))
        gn = torch.stack(torch._foreach_norm([st.flat_grad[s:s + n] for s, n in views]))
        wd = self.group_hyper[self._lars_group, 2]
        trust = torch.where(self._lars_flag & (wn > 0) & (gn > 0),
                            self.trust_coefficient * wn / (gn + wd * wn + LARS_EPS), torch.ones_like(wn))
        k = 0
        for b in st.buckets:
            if b.lars:
                b.trust.copy_(trust[k:k + len(b.params)])
            k += len(b.params)
        return torch.cat([trust, trust.new_ones(1)])[self._lars_index].unsqueeze(1)

    # ----------------------------------------------------------- step --
    def _fwd_bwd(self, x, y):
        st = self.state
        if not self._carry:  # gradients of a preceding no_sync() step are kept and added to
            st.zero_grad()
        for b in st.buckets:
            b.pending = len(b.params)
        import contextlib
        with (fused_bn.defer_counters() if self._defer_nbt else contextlib.nullcontext()) as counters, nvtx.range("b200mpi.forward"):
            if self.autocast_dtype is not None:
                with torch.autocast(self.device.type, dtype=self.autocast_dtype):
                    out = self.model(x)
                    loss = self.loss_fn(out, y)
            else:
                loss = self.loss_fn(self.model(x), y)
        if counters:   # one multi-tensor add instead of one tiny kernel per BN layer
            torch._foreach_add_(counters, 1)
        if self._sync and self._ema_sched is not None:   # k of this update; the bucket kernels read it after the main->comm event
            self._ema_sched[1:].add_(1)
        if self._sync and self.lr_schedule is not None:  # this update's rates, read the same way
            self._schedule_step()
        with nvtx.range("b200mpi.backward+allreduce_sgd"):   # bucket kernels are launched from the autograd hooks inside
            loss.backward()
        self._loss.copy_(loss.detach())
        if not self._sync:   # local accumulation only (Horovod: backward_passes_per_step > 1)
            self._carry = True
            return
        for b in st.buckets:  # parameters that received no gradient this step
            if b.pending != -1:
                self._reduce_bucket(b)
        if self._cuda:
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
        if not self.fused:
            self._unfused_sgd()
            if self._flat_ema is not None:
                self._unfused_ema()
        self._carry = False

    def _ensure_static(self, x, y):
        if self._static_x is None or self._static_x.shape != x.shape:
            self._static_x = torch.empty(x.shape, dtype=x.dtype, device=self.device)
            if self.channels_last and x.dim() == 4:
                self._static_x = self._static_x.contiguous(memory_format=torch.channels_last)
            self._static_y = torch.empty(y.shape, dtype=y.dtype, device=self.device)
            self._graph = None

    # ------------------------------------------------- input pipeline --
    def prefetch(self, x, y) -> None:
        """Start moving the NEXT batch to the device now (``async_h2d`` mode: on a copy stream, into one of two staging
        buffers, overlapping whatever the compute stream is still doing); the following ``step()`` without arguments
        trains on it. A loop that reads the loss every step keeps the copy off the critical path with

            trainer.prefetch(x0, y0)
            for i in range(n):
                loss = trainer.step()                 # enqueue step i (inputs already on their way)
                trainer.prefetch(x[i + 1], y[i + 1])  # H2D of the next batch runs under step i
                print(float(loss))                    # only now wait for step i
        """
        self._ensure_static(x, y)
        if not (self.async_h2d and self._cuda):
            self._pending_batch = (x, y)
            return
        if self._stage_x is None or self._stage_x[0].shape != x.shape or self._stage_x[0].dtype != x.dtype:
            # staging buffers keep the HOST layout, so the H2D copy is one plain DMA; the layout change to channels-last
            # happens in the device-to-device copy into the graph's static input
            self._stage_x = [torch.empty(x.shape, dtype=x.dtype, device=self.device) for _ in range(2)]
            self._stage_y = [torch.empty(y.shape, dtype=y.dtype, device=self.device) for _ in range(2)]
            self._stage_ready = [torch.cuda.Event() for _ in range(2)]
            self._stage_free = [torch.cuda.Event() for _ in range(2)]
            for ev in self._stage_free:
                ev.record(torch.cuda.current_stream(self.device))
            self._stage_idx = 0
        k = self._stage_idx
        self._stage_idx ^= 1
        cs = self._copy_stream
        cs.wait_event(self._stage_free[k])       # buffer k was last read by the D2D copy two steps ago
        with torch.cuda.stream(cs):
            self._stage_x[k].copy_(x, non_blocking=True)
            self._stage_y[k].copy_(y, non_blocking=True)
            self._stage_ready[k].record(cs)
        self._pending_batch = k

    def _consume_batch(self) -> None:
        """Make the prefetched batch the graph's static input (main stream)."""
        pb, self._pending_batch = self._pending_batch, None
        if pb is None:
            raise RuntimeError("step() without arguments needs a prefetch() first")
        if isinstance(pb, tuple):                 # synchronous mode: the copy happens here, on the compute stream
            self._static_x.copy_(pb[0], non_blocking=True)
            self._static_y.copy_(pb[1], non_blocking=True)
            return
        main = torch.cuda.current_stream(self.device)
        main.wait_event(self._stage_ready[pb])
        self._static_x.copy_(self._stage_x[pb], non_blocking=True)
        self._static_y.copy_(self._stage_y[pb], non_blocking=True)
        self._stage_free[pb].record(main)

    def step(self, x=None, y=None):
        """One optimizer step on a batch given as (pinned) host or device tensors; without arguments, on the batch handed
        to ``prefetch()``. Returns the loss as a device scalar (``float(loss)`` is the D2H read)."""
        if self._in_ema:
            raise RuntimeError("step() inside ema_weights(): the parameter window holds the averaged weights")
        self._fault.on_step()
        if x is not None:
            self.prefetch(x, y)
        self._consume_batch()
        if not self.use_graph or not self._cuda or not self._sync or self._carry:
            n0 = self.comm.launch_count + fused_bn.launch_count()
            self._fwd_bwd(self._static_x, self._static_y)
            self._launches_per_step = self.comm.launch_count + fused_bn.launch_count() - n0
            return self._loss
        if self._graph is None:
            self._capture()
        self._graph.replay()
        self._replays += 1
        return self._loss

    def _capture(self):
        # warm up eagerly on a side stream (cuDNN autotune, allocator) before capture
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(3):
                self._fwd_bwd(self._static_x, self._static_y)
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        if self.comm.world > 1:
            self.comm.host_barrier()
        g = torch.cuda.CUDAGraph()
        n0 = self.comm.launch_count + fused_bn.launch_count()
        before = {(o["op"], o["algo"]): o for o in self.comm.stats(native_only=True)["ops"]} if hasattr(self.comm, "stats") else {}
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            self._fwd_bwd(self._static_x, self._static_y)
        self._launches_per_step = self.comm.launch_count + fused_bn.launch_count() - n0   # our kernels in one replay
        if hasattr(self.comm, "stats"):
            self._folded_ops = self._replayed_ops()
            self._graph_ops, self._replays = [], 0
            for o in self.comm.stats(native_only=True)["ops"]:
                b = before.get((o["op"], o["algo"]), {"calls": 0, "bytes": 0})
                if o["calls"] > b["calls"]:
                    self._graph_ops.append({"op": o["op"], "algo": o["algo"], "calls": o["calls"] - b["calls"],
                                            "bytes": o["bytes"] - b["bytes"]})
        self._graph = g
        torch.cuda.synchronize(self.device)
        if self.comm.world > 1:
            self.comm.host_barrier()

    # ---------------------------------------------------------- evaluation --
    MAX_EVAL_GRAPHS = 2   # e.g. the full batch and a ragged last batch; further shapes run eagerly

    def _eval_stats(self, x, y, topk):
        """Eval-mode forward, loss and top-k hits packed into one vector ``[loss, hits@k / n ...]``; returns (vector, ks)."""
        if self.autocast_dtype is not None:
            with torch.autocast(self.device.type, dtype=self.autocast_dtype):
                out = self.model(x)
                loss = self.loss_fn(out, y)
        else:
            out = self.model(x)
            loss = self.loss_fn(out, y)
        ks = [k for k in topk if k <= out.shape[1]]
        top = out.float().topk(max(ks), dim=1).indices if ks else None
        stats = [loss.float().reshape(())] + [(top[:, :k] == y[:, None]).any(1).float().mean() for k in ks]
        return torch.stack(stats).contiguous(), ks

    def _eval_graph(self, x, y, topk):
        """The eval graph for this input shape, captured on first use (at most MAX_EVAL_GRAPHS; None: run eagerly). Each has
        its own static inputs and memory pool; replays read the live parameters and running statistics, which training updates
        in place, so a graph stays valid across steps. Capture uses the eval kernels only: nothing the training step owns
        (its graph, static buffers, BN workspace, running statistics) is written."""
        key = (tuple(x.shape), x.dtype, tuple(y.shape), y.dtype, tuple(topk))
        ent = self._eval_graphs.get(key)
        if ent is not None or len(self._eval_graphs) >= self.MAX_EVAL_GRAPHS:
            return ent
        sx = torch.empty(x.shape, dtype=x.dtype, device=self.device)
        if self.channels_last and x.dim() == 4:
            sx = sx.contiguous(memory_format=torch.channels_last)
        sy = torch.empty(y.shape, dtype=y.dtype, device=self.device)
        sx.copy_(x)
        sy.copy_(y)
        s = torch.cuda.Stream(device=self.device)   # warm up eagerly first (cuDNN algorithm choice, allocator)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            self._eval_stats(sx, sy, topk)
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            vec, ks = self._eval_stats(sx, sy, topk)
        ent = self._eval_graphs[key] = (g, sx, sy, vec, ks)
        return ent

    @torch.no_grad()
    def evaluate(self, x, y, topk=(1, 5)):
        """Forward only, in eval mode (BatchNorm uses its running statistics), under the trainer's autocast setting; no gradient,
        no collective on the training path, the captured CUDA graph is left alone. Returns ``{"loss": ..., "top1": ..., "top5": ...,
        "examples": n}`` averaged over the ranks (tf_cnn_benchmarks' ``--eval``: "Accuracy @ 1 / @ 5").

        With ``cuda_graph`` on CUDA the forward, loss and top-k run as one graph replay per call (one graph per input shape,
        at most MAX_EVAL_GRAPHS); the average over the ranks stays an eager collective after it."""
        was_training = self.model.training
        self.model.eval()
        try:
            ent = self._eval_graph(x, y, topk) if (self.use_graph and self._cuda) else None
            if ent is not None:
                g, sx, sy, out_vec, ks = ent
                sx.copy_(x, non_blocking=True)
                sy.copy_(y, non_blocking=True)
                g.replay()
                vec = out_vec.clone()
            else:
                x = x.to(self.device, non_blocking=True)
                y = y.to(self.device, non_blocking=True)
                if self.channels_last and x.dim() == 4:
                    x = x.contiguous(memory_format=torch.channels_last)
                vec, ks = self._eval_stats(x, y, topk)
            if self.comm.world > 1:
                self.comm.allreduce(vec, op="avg")
            vals = vec.tolist()
            res = {"loss": vals[0], "examples": int(y.shape[0]) * self.comm.world}
            for k, v in zip(ks, vals[1:]):
                res[f"top{k}"] = v
            return res
        finally:
            self.model.train(was_training)

    # ------------------------------------------------- checkpoint / resume --
    def state_dict(self) -> dict:
        """World-size independent checkpoint of the training state (SURVEY.md section 5.4; the reference's examples checkpoint on
        rank 0 only, tensorflow_mnist.py:159): fp32 MASTER parameters, module buffers (BN running statistics), the optimizer's
        momentum and the hyper-parameters, all keyed by parameter / buffer NAME and moved to the host. COLLECTIVE when
        world > 1: the fused optimizer keeps only 1/world of every bucket's momentum on each rank, so the shards are
        all-gathered first (one byte-wise allgather kernel per bucket); every rank gets the full dictionary, write it from rank 0.
        Loading re-shards for whatever world the new trainer runs in (elastic rescale, different GPU count)."""
        if self._in_ema:
            raise RuntimeError("state_dict() inside ema_weights(): the parameter window holds the averaged weights")
        st = self.state
        names = {p: n for n, p in self.model.named_parameters()}
        if self._cuda:
            torch.cuda.synchronize(self.device)
        mom_flat = torch.zeros(st.total, dtype=torch.float32, device=st.flat_param.device)
        if self.fused:
            mom_flat = self._gather_shards("momentum")
        elif hasattr(self, "_flat_mom"):
            mom_flat.copy_(self._flat_mom)
        masters, momentum = {}, {}
        for p in st.params:
            start, n = st.param_slot[p][1], p.numel()
            masters[names[p]] = st.flat_param[start:start + n].as_strided(p.size(), p.stride()).detach().cpu().contiguous()
            momentum[names[p]] = mom_flat[start:start + n].as_strided(p.size(), p.stride()).detach().cpu().contiguous()
        sd = {"format": "b200mpi.DataParallelTrainer/1", "model": masters, "momentum": momentum,
              "buffers": {n: b.detach().cpu().clone() for n, b in self.model.named_buffers()},
              "hyper": {"lr": float(self.hyper[0]) if self.lr_schedule is None else float(self._lr), "momentum": float(self.hyper[1]), "weight_decay": float(self.hyper[2]),
                        "nesterov": bool(self.nesterov), "lars": bool(self._group_lars[0]),
                        "trust_coefficient": self.trust_coefficient},
              "world_size_at_save": int(self.comm.world)}
        if self._has_groups:
            sd["param_groups"] = self.param_groups
        if self.ema_decay is not None:
            ema_flat = self._gather_ema()
            sd["ema"] = {names[p]: ema_flat[st.param_slot[p][1]:st.param_slot[p][1] + p.numel()].as_strided(p.size(), p.stride())
                         .detach().cpu().contiguous() for p in st.params}
            sd["ema_updates"] = self.ema_updates
            sd["hyper"]["ema_decay"] = self.ema_decay
        if self.lr_schedule is not None:
            sd["lr_schedule"] = self.lr_schedule.to_dict()
            sd["lr_schedule_step"] = self.lr_schedule_step
        return sd

    def _gather_shards(self, attr: str) -> torch.Tensor:
        """The full flat fp32 buffer of a per-bucket sharded state (``"momentum"`` or ``"ema"``); one allgather per bucket,
        COLLECTIVE when world > 1."""
        st = self.state
        out = torch.zeros(st.total, dtype=torch.float32, device=st.flat_param.device)
        W = self.comm.world
        for b in st.buckets:
            shard = getattr(b, attr)
            full = shard
            if W > 1:
                full = torch.empty(W * shard.numel(), dtype=torch.float32, device=shard.device)
                self.comm.allgather(shard, full)
            out[b.start:b.start + b.numel] = full[:b.numel]
        if self._cuda:
            torch.cuda.synchronize(self.device)
        return out

    def _gather_ema(self) -> torch.Tensor:
        """The weight average as one full flat fp32 buffer (COLLECTIVE on the fused path when world > 1)."""
        if self._cuda:
            torch.cuda.synchronize(self.device)
        return self._gather_shards("ema") if self.fused else self._flat_ema.clone()

    def _set_ema(self, flat: torch.Tensor) -> None:
        """Make the weight average ``flat`` (a full flat fp32 buffer): this rank's shard of every bucket, or the flat copy."""
        st = self.state
        if not self.fused:
            # in place once it exists: a captured graph (comm_backend="nccl") keeps updating this buffer
            if self._flat_ema is None:
                self._flat_ema = flat.detach().clone()
            else:
                self._flat_ema.copy_(flat)
            return
        r = self.comm.rank
        for b in st.buckets:
            per = b.ema.numel()
            lo, hi = min(r * per, b.numel), min((r + 1) * per, b.numel)
            b.ema.zero_()
            b.ema[:hi - lo] = flat[b.start + lo:b.start + hi]

    @property
    def ema_updates(self) -> int:
        """k: the number of parameter updates the weight average has seen (reading it synchronises with the device)."""
        return int(self._ema_sched[1]) if self._ema_sched is not None else 0

    @contextlib.contextmanager
    def ema_weights(self):
        """Context manager: inside it the model's parameters (fp32 masters and the bf16 shadow) hold the weight average, so
        ``evaluate()`` (its CUDA graphs included) runs on the averaged weights with the live BatchNorm statistics; on exit the
        trained parameters are restored bit for bit. ``step()`` and ``state_dict()`` inside it raise ``RuntimeError``.
        COLLECTIVE when world > 1 (the shards are all-gathered on entry)."""
        if self.ema_decay is None:
            raise RuntimeError("ema_weights() needs a trainer built with ema_decay")
        if self._in_ema:
            raise RuntimeError("ema_weights() is already active")
        st = self.state
        ema_flat = self._gather_ema()
        with torch.no_grad():
            saved = st.flat_param.clone()
            st.flat_param.copy_(ema_flat)
            st.refresh_lowp()
        self._in_ema = True
        try:
            yield self
        finally:
            with torch.no_grad():
                st.flat_param.copy_(saved)
                st.refresh_lowp()
            self._in_ema = False
            if self._cuda:
                torch.cuda.synchronize(self.device)

    def load_state_dict(self, sd: dict, load_hyper: bool = True) -> None:
        """Restore ``state_dict()`` output in a trainer built on the same model class (any world size, with or without the bf16
        shadow / fused optimizer). Not collective: every rank loads the same dictionary and keeps its own momentum shard.
        With ``load_hyper``, per-group values are restored when the checkpoint's parameter groups have the same members (by
        name) as this trainer's; a checkpoint with groups into a trainer without them, or the reverse, is a ``ValueError``.
        Which groups use LARS and ``trust_coefficient`` stay as this trainer was built (the checkpoint records them): the
        momentum is the same state for SGD and LARS, so SGD and LARS checkpoints load into each other. With ``ema_decay`` the
        weight average and its update count are restored from ``"ema"`` / ``"ema_updates"``, or, for a checkpoint without
        them, restart from the loaded parameters at count 0; the decay stays this trainer's. Without ``ema_decay`` they are
        ignored. With ``lr_schedule`` the step count comes back from ``"lr_schedule_step"`` (0 when absent), the loaded
        ``lr`` values are the base rates and the schedule stays this trainer's; without it both keys are ignored."""
        if self._in_ema:
            raise RuntimeError("load_state_dict() inside ema_weights(): leaving the context would undo it")
        if sd.get("format") != "b200mpi.DataParallelTrainer/1":
            raise ValueError("not a DataParallelTrainer checkpoint")
        if load_hyper and ("param_groups" in sd) != self._has_groups:
            raise ValueError("parameter groups: the checkpoint has them and this trainer does not, or the reverse "
                             "(load_hyper=False skips the hyper-parameters)")
        if load_hyper and self._has_groups:
            theirs = [sorted(g["params"]) for g in sd["param_groups"]]
            if theirs != [sorted(n) for n in self._group_names]:
                raise ValueError("parameter groups of the checkpoint have other members than this trainer's")
        st = self.state
        names = {p: n for n, p in self.model.named_parameters()}
        missing = [n for n in names.values() if n not in sd["model"]]
        if missing:
            raise KeyError(f"checkpoint lacks parameters {missing[:5]}{' ...' if len(missing) > 5 else ''}")
        dev = st.flat_param.device
        mom_flat = torch.zeros(st.total, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for p in st.params:
                start, n, name = st.param_slot[p][1], p.numel(), names[p]
                src = sd["model"][name]
                if tuple(src.shape) != tuple(p.shape):
                    raise ValueError(f"shape of {name}: checkpoint {tuple(src.shape)} vs model {tuple(p.shape)}")
                st.flat_param[start:start + n].as_strided(p.size(), p.stride()).copy_(src.to(dev, torch.float32))
                if name in sd.get("momentum", {}):
                    mom_flat[start:start + n].as_strided(p.size(), p.stride()).copy_(sd["momentum"][name].to(dev, torch.float32))
            st.refresh_lowp()
            bufs = dict(self.model.named_buffers())
            for n, b in sd.get("buffers", {}).items():
                if n in bufs:
                    bufs[n].copy_(b.to(bufs[n].device, bufs[n].dtype))
            if self.fused:
                r = self.comm.rank
                for b in st.buckets:
                    per = b.momentum.numel()
                    lo, hi = min(r * per, b.numel), min((r + 1) * per, b.numel)
                    b.momentum.zero_()
                    b.momentum[:hi - lo] = mom_flat[b.start + lo:b.start + hi]
            else:
                self._flat_mom = mom_flat
            if self.ema_decay is not None:
                ema_flat = st.flat_param.clone()
                for p in st.params:
                    name = names[p]
                    if name in sd.get("ema", {}):
                        start, n = st.param_slot[p][1], p.numel()
                        ema_flat[start:start + n].as_strided(p.size(), p.stride()).copy_(sd["ema"][name].to(dev, torch.float32))
                self._set_ema(ema_flat)
                self._ema_sched[1] = float(sd.get("ema_updates", 0)) if "ema" in sd else 0.0
        if load_hyper and "hyper" in sd:
            h = sd["hyper"]
            self._lr, self._mu, self._wd = h["lr"], h["momentum"], h["weight_decay"]
            self.hyper.copy_(torch.tensor([self._lr, self._mu, self._wd], dtype=torch.float32))
            self._group_vals[0] = [self._lr, self._mu, self._wd]
            if self.group_hyper is not None and not self._has_groups:   # LARS without param_groups: its one-row table
                self.group_hyper[0].copy_(self.hyper)
            if self._has_groups:
                self._group_vals = [[g["lr"], g["momentum"], g["weight_decay"]] for g in sd["param_groups"]]
                self.group_hyper.copy_(torch.tensor(self._group_vals, dtype=torch.float32))
        if self.lr_schedule is not None:
            k = int(sd.get("lr_schedule_step", 0))
            if k < 0:
                raise ValueError(f"lr_schedule_step must be >= 0, got {k}")
            self._lr_base.copy_(torch.tensor([float(v[0]) for v in self._group_vals], dtype=torch.float64))
            self._lr_step.fill_(k)
            if k > 0:   # the tables hold what the last step used, as after that step
                self._write_rates(k - 1)
        if self._cuda:
            torch.cuda.synchronize(self.device)

    def no_sync(self):
        """Context manager: steps inside accumulate gradients locally (no collective, no update, run eagerly);
        the first step after it reduces the accumulated sum and applies one update."""
        trainer = self

        class _Ctx:
            def __enter__(self_inner):
                trainer._sync = False

            def __exit__(self_inner, *exc):
                trainer._sync = True
        return _Ctx()
