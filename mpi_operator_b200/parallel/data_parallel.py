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

import os
from dataclasses import dataclass, field
from typing import Callable, List, Optional

import torch
import torch.nn as nn

from ..ops import fused_bn
from ..runtime.comm import Communicator, Window
from ..utils import fault, nvtx


def _align(n: int, a: int) -> int:
    return (n + a - 1) // a * a


@dataclass
class Bucket:
    index: int
    start: int            # element offset in the flat buffers
    numel: int            # padded to a multiple of 8 elements (16-byte vectors for fp32 and bf16)
    params: List[nn.Parameter] = field(default_factory=list)
    pending: int = 0
    momentum: Optional[torch.Tensor] = None  # this rank's shard


class FlatModelState:
    """Re-homes a module's parameters and gradients into two symmetric windows
    with identical element layout (fp32), bucketed in reverse registration order
    (the order backward produces them).

    ``bf16_params=True`` adds a third window with the same element layout in bf16: matrix-shaped
    parameters (conv / linear weights) become bf16 leaves that view it, their fp32 masters stay in
    the parameter window and the fused SGD kernel refreshes the shadow in the same pass
    (``lowp_win``). Forward then needs no per-layer fp32->bf16 weight cast and backward no
    bf16->fp32 gradient cast + accumulate: ~3 small kernels per layer disappear from the step."""

    def __init__(self, module: nn.Module, comm: Communicator, bucket_bytes: int = 32 << 20, bf16_params: bool = False):
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
    """

    def __init__(self, model: nn.Module, loss_fn: Callable, comm: Communicator, *, lr: float, momentum: float = 0.9,
                 weight_decay: float = 0.0, nesterov: bool = False, bucket_bytes: Optional[int] = None,
                 autocast_dtype: Optional[torch.dtype] = torch.bfloat16, channels_last: bool = True,
                 cuda_graph: bool = True, fused_optimizer: bool = True, algo: Optional[str] = None,
                 comm_backend: str = "b200mpi", bf16_params: Optional[bool] = None, async_h2d: Optional[bool] = None):
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
        self.state = FlatModelState(model, comm, bucket_bytes, bf16_params=self.bf16_params)
        self.state.broadcast_parameters(0)
        # {lr, momentum, weight_decay} on the device: graph replays follow schedules
        self.hyper = torch.tensor([lr, momentum, weight_decay], device=self.device, dtype=torch.float32)
        comm.set_hyper(self.hyper)
        self._lr, self._mu, self._wd = lr, momentum, weight_decay
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
    def set_lr(self, lr: float) -> None:
        self._lr = lr
        self.hyper[0] = lr

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
        if self.backend == "nccl":
            g = st.flat_grad[b.start:b.start + b.numel]
            if self.comm.world > 1:
                self._dist.all_reduce(g, op=self._dist.ReduceOp.AVG)
        elif self.fused:
            self.comm.allreduce_sgd_window(st.grad_win, b.start * 4, st.param_win, b.start * 4, b.momentum,
                                           b.numel, torch.float32, lr=self._lr, momentum_coef=self._mu,
                                           weight_decay=self._wd, nesterov=self.nesterov,
                                           lowp_win=st.lowp_win, lowp_off=b.start * 2, algo=self.algo,
                                           stream=self.comm_stream)
        else:
            self.comm.allreduce_window(st.grad_win, b.start * 4, b.numel, torch.float32, op="avg",
                                       algo=self.algo, stream=self.comm_stream)

    def _unfused_sgd(self) -> None:
        """Plain flat SGD (used by the NCCL baseline and fused_optimizer=False)."""
        st = self.state
        if not hasattr(self, "_flat_mom"):
            self._flat_mom = torch.zeros_like(st.flat_param)
        g = st.flat_grad
        if self._wd:
            g = g.add(st.flat_param, alpha=self._wd)
        self._flat_mom.mul_(self.hyper[1]).add_(g)
        upd = g.add(self._flat_mom, alpha=self._mu) if self.nesterov else self._flat_mom
        st.flat_param.sub_(upd * self.hyper[0])
        st.refresh_lowp()

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
    @torch.no_grad()
    def evaluate(self, x, y, topk=(1, 5)):
        """Forward only, in eval mode (BatchNorm uses its running statistics), under the trainer's autocast setting; no gradient,
        no collective on the training path, the captured CUDA graph is left alone. Returns ``{"loss": ..., "top1": ..., "top5": ...,
        "examples": n}`` averaged over the ranks (tf_cnn_benchmarks' ``--eval``: "Accuracy @ 1 / @ 5")."""
        was_training = self.model.training
        self.model.eval()
        try:
            x = x.to(self.device, non_blocking=True)
            y = y.to(self.device, non_blocking=True)
            if self.channels_last and x.dim() == 4:
                x = x.contiguous(memory_format=torch.channels_last)
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
            vec = torch.stack(stats).contiguous()
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
        st = self.state
        names = {p: n for n, p in self.model.named_parameters()}
        if self._cuda:
            torch.cuda.synchronize(self.device)
        mom_flat = torch.zeros(st.total, dtype=torch.float32, device=st.flat_param.device)
        if self.fused:
            W = self.comm.world
            for b in st.buckets:
                per = b.momentum.numel()
                full = b.momentum
                if W > 1:
                    full = torch.empty(W * per, dtype=torch.float32, device=b.momentum.device)
                    self.comm.allgather(b.momentum, full)
                mom_flat[b.start:b.start + b.numel] = full[:b.numel]
            if self._cuda:
                torch.cuda.synchronize(self.device)
        elif hasattr(self, "_flat_mom"):
            mom_flat.copy_(self._flat_mom)
        masters, momentum = {}, {}
        for p in st.params:
            start, n = st.param_slot[p][1], p.numel()
            masters[names[p]] = st.flat_param[start:start + n].as_strided(p.size(), p.stride()).detach().cpu().contiguous()
            momentum[names[p]] = mom_flat[start:start + n].as_strided(p.size(), p.stride()).detach().cpu().contiguous()
        return {"format": "b200mpi.DataParallelTrainer/1", "model": masters, "momentum": momentum,
                "buffers": {n: b.detach().cpu().clone() for n, b in self.model.named_buffers()},
                "hyper": {"lr": float(self.hyper[0]), "momentum": float(self.hyper[1]), "weight_decay": float(self.hyper[2]),
                          "nesterov": bool(self.nesterov)},
                "world_size_at_save": int(self.comm.world)}

    def load_state_dict(self, sd: dict, load_hyper: bool = True) -> None:
        """Restore ``state_dict()`` output in a trainer built on the same model class (any world size, with or without the bf16
        shadow / fused optimizer). Not collective: every rank loads the same dictionary and keeps its own momentum shard."""
        if sd.get("format") != "b200mpi.DataParallelTrainer/1":
            raise ValueError("not a DataParallelTrainer checkpoint")
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
        if load_hyper and "hyper" in sd:
            h = sd["hyper"]
            self._lr, self._mu, self._wd = h["lr"], h["momentum"], h["weight_decay"]
            self.hyper.copy_(torch.tensor([self._lr, self._mu, self._wd], dtype=torch.float32))
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
