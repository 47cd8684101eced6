#!/usr/bin/env python
"""tf_cnn_benchmarks-compatible entry point (same path + flags as the command in the
reference's headline MPIJob: examples/v2beta1/tensorflow-benchmarks/
tensorflow-benchmarks.yaml:38-42  ``python scripts/tf_cnn_benchmarks/
tf_cnn_benchmarks.py --model=resnet101 --batch_size=64 --variable_update=horovod``).

The reference image clones tensorflow/benchmarks (TF1 + Horovod + NCCL); here the
same flags drive the PyTorch + b200mpi stack: synthetic ImageNet, SGD momentum,
NCHW logical layout (channels_last memory), bf16 autocast, and the log format of
the reference's sample output (README.md:180-212): a line every 10 steps and a
final ``total images/sec``.
"""
import argparse
import contextlib
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..", "..", "..")))


def main():
    ap = argparse.ArgumentParser(allow_abbrev=False)
    ap.add_argument("--model", default="resnet50")
    ap.add_argument("--batch_size", type=int, default=64, help="per device")
    ap.add_argument("--variable_update", default="horovod", choices=["horovod", "replicated", "parameter_server", "independent"])
    ap.add_argument("--num_batches", type=int, default=100)
    ap.add_argument("--num_warmup_batches", type=int, default=10)
    ap.add_argument("--display_every", type=int, default=10)
    ap.add_argument("--optimizer", default="sgd", choices=["sgd", "momentum"])
    ap.add_argument("--init_learning_rate", type=float, default=0.01)
    ap.add_argument("--momentum", type=float, default=0.9)
    ap.add_argument("--weight_decay", type=float, default=0.0)
    ap.add_argument("--use_fp16", default="False")
    ap.add_argument("--data_format", default="NCHW")
    ap.add_argument("--data_name", default="imagenet")
    ap.add_argument("--device", default="gpu", choices=["gpu", "cpu"], help="cpu: host tensors through the Horovod-API engine (no CUDA needed)")
    ap.add_argument("--image_size", type=int, default=224)
    ap.add_argument("--num_gpus", type=int, default=1)
    ap.add_argument("--eval", default="False", help="tf_cnn_benchmarks flag: evaluate (forward only) instead of training; restores --train_dir")
    ap.add_argument("--train_dir", default="", help="checkpoint directory (tf_cnn_benchmarks flag): restored from at start if it holds a "
                                                    "checkpoint, written by rank 0 at the end")
    ap.add_argument("--moving_average_decay", type=float, default=0.0,
                    help="tf_cnn_benchmarks flag: keep an exponential moving average of the weights with this decay (0: off); "
                         "--eval evaluates the averaged weights")
    ap.add_argument("--piecewise_learning_rate_schedule", default="",
                    help='tf_cnn_benchmarks flag: "v0;e1;v1;e2;v2;..." - learning rate v0 until epoch e1, v1 until e2, ...; '
                         "takes precedence over --init_learning_rate")
    ap.add_argument("--num_learning_rate_warmup_epochs", type=float, default=0.0,
                    help="tf_cnn_benchmarks flag: ramp the learning rate linearly from 0 over this many epochs")
    ap.add_argument("--num_epochs_per_decay", type=float, default=0.0,
                    help="tf_cnn_benchmarks flag: with --learning_rate_decay_factor, multiply the learning rate by the factor "
                         "every this many epochs (staircase)")
    ap.add_argument("--learning_rate_decay_factor", type=float, default=0.0, help="tf_cnn_benchmarks flag: see --num_epochs_per_decay")
    ap.add_argument("--minimum_learning_rate", type=float, default=0.0,
                    help="tf_cnn_benchmarks flag: lower bound of the exponentially decayed learning rate")
    ap.add_argument("--b200_engine", default=os.environ.get("B200MPI_ENGINE", "fused"), choices=["fused", "hvd", "nccl"],
                    help="fused: symmetric-window grads + fused allreduce+SGD kernel in a CUDA graph; "
                         "hvd: hvd.DistributedOptimizer API path; nccl: stock NCCL baseline")
    ap.add_argument("--b200_compute_dtype", default="bf16", choices=["bf16", "fp32"])
    args, unknown = ap.parse_known_args()
    if unknown:
        print(f"tf_cnn_benchmarks (b200): ignoring flags {unknown}", file=sys.stderr)

    import torch
    import torch.nn as nn
    import mpi_operator_b200.hvd as hvd
    from mpi_operator_b200.models import build_model
    from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
    from mpi_operator_b200.parallel.lr_schedule import LRSchedule

    hvd.init()
    rank, size = hvd.rank(), hvd.size()
    on_gpu = args.device == "gpu"
    if on_gpu and not torch.cuda.is_available():
        raise SystemExit("tf_cnn_benchmarks (b200): --device=gpu but no CUDA device is visible (use --device=cpu for a host run)")
    evaluating = str(args.eval).lower() == "true"
    averaging = args.moving_average_decay != 0.0
    if not on_gpu:   # host run: the Horovod-API engine, except for --eval and the weight average, which need the trainer (then
        # with the unfused optimizer)
        args.b200_engine, args.b200_compute_dtype = ("fused" if (evaluating or averaging) else "hvd"), "fp32"
    if averaging and args.b200_engine not in ("fused", "nccl"):
        raise SystemExit("tf_cnn_benchmarks (b200): --moving_average_decay needs the trainer engines (fused | nccl)")
    S = args.image_size
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(1234 + rank)
    mu = args.momentum if args.optimizer == "momentum" or args.momentum else 0.0
    lr = args.init_learning_rate * size  # Horovod convention (tensorflow_mnist.py:123-130)
    B = args.batch_size
    # learning-rate schedule, tf_cnn_benchmarks' get_learning_rate: epochs count images of the global batch, every rate is
    # scaled by the world size like --init_learning_rate, and the warm-up ramps to the first rate
    steps_per_epoch = 1281167.0 / (B * size)
    warmup = int(steps_per_epoch * args.num_learning_rate_warmup_epochs) if args.num_learning_rate_warmup_epochs > 0 else 0
    lr_schedule = None
    try:
        if args.piecewise_learning_rate_schedule:
            parts = args.piecewise_learning_rate_schedule.split(";")
            vals, epochs = [float(v) for v in parts[0::2]], [float(e) for e in parts[1::2]]
            if len(parts) % 2 != 1 or not vals[0] > 0:
                raise ValueError("--piecewise_learning_rate_schedule needs 'v0;e1;v1;...' with v0 > 0")
            lr = vals[0] * size
            lr_schedule = LRSchedule.piecewise([int(steps_per_epoch * e) for e in epochs], [v / vals[0] for v in vals],
                                               warmup_steps=warmup)
        elif args.num_epochs_per_decay > 0 and args.learning_rate_decay_factor > 0:
            if not args.init_learning_rate > 0:
                raise ValueError("exponential decay needs --init_learning_rate > 0")
            lr_schedule = LRSchedule.exponential(int(steps_per_epoch * args.num_epochs_per_decay), args.learning_rate_decay_factor,
                                                 floor=args.minimum_learning_rate / args.init_learning_rate, warmup_steps=warmup)
        elif warmup:
            lr_schedule = LRSchedule.constant(warmup_steps=warmup)
    except ValueError as e:
        raise SystemExit(f"tf_cnn_benchmarks (b200): learning-rate schedule: {e}")
    model = build_model(args.model, **({"image_size": S} if args.model == "trivial" else {}))
    loss_fn = nn.CrossEntropyLoss()
    dtype = torch.bfloat16 if on_gpu and (args.b200_compute_dtype == "bf16" or str(args.use_fp16).lower() == "true") else None
    x = torch.randn(B, 3, S, S)
    y = torch.randint(0, 1000, (B,))
    if on_gpu:
        x, y = x.pin_memory(), y.pin_memory()

    if rank == 0:
        print("TensorFlow:  n/a (PyTorch %s + b200mpi runtime)" % torch.__version__)
        print(f"Model:       {args.model}")
        print(f"Dataset:     {args.data_name} (synthetic)")
        print("Mode:        training")
        print("SingleSess:  False")
        print(f"Batch size:  {B * size} global")
        print(f"             {B} per device")
        print(f"Num batches: {args.num_batches}")
        print("Num epochs:  %.2f" % (args.num_batches * B * size / 1281167.0))
        print(f"Devices:     {['horovod/%s:%d' % (args.device, i) for i in range(size)]}")
        print(f"Data format: {args.data_format}")
        print(f"Optimizer:   {args.optimizer}")
        print(f"LR:          {lr:g}" + (f" x {lr_schedule!r}" if lr_schedule is not None else ""))
        print(f"Variables:   {args.variable_update}")
        print(f"Engine:      {args.b200_engine} (NVLS multicast: {getattr(hvd._comm(), 'has_multicast', False)})")
        print("==========")
        print("Generating model")
        sys.stdout.flush()

    if args.b200_engine in ("fused", "nccl"):
        if args.b200_engine == "nccl" and size > 1:
            import torch.distributed as dist
            dist.init_process_group("nccl", rank=rank, world_size=size, device_id=torch.device("cuda", torch.cuda.current_device()))
        trainer = DataParallelTrainer(model, loss_fn, hvd._comm(), lr=lr, momentum=mu, weight_decay=args.weight_decay,
                                      autocast_dtype=dtype, comm_backend="nccl" if args.b200_engine == "nccl" else "b200mpi",
                                      fused_optimizer=on_gpu, cuda_graph=on_gpu,
                                      ema_decay=args.moving_average_decay if averaging else None, lr_schedule=lr_schedule)

        def step():
            return trainer.step(x, y)
    else:
        dev = "cuda" if on_gpu else "cpu"
        model = model.to(dev).to(memory_format=torch.channels_last)
        sgd = torch.optim.SGD(model.parameters(), lr=lr, momentum=mu, weight_decay=args.weight_decay)
        opt = hvd.DistributedOptimizer(sgd, named_parameters=model.named_parameters(), op=hvd.Average)
        lr_sched = None   # a LambdaLR over the same multiplier, made once the resumed step count is known
        hvd.broadcast_parameters(model.state_dict(), root_rank=0)
        sx = torch.empty(B, 3, S, S, device=dev).contiguous(memory_format=torch.channels_last)
        sy = torch.empty(B, dtype=torch.long, device=dev)

        def step():
            sx.copy_(x, non_blocking=True)
            sy.copy_(y, non_blocking=True)
            opt.zero_grad()
            with torch.autocast(dev, dtype=dtype, enabled=dtype is not None):
                loss = loss_fn(model(sx), sy)
            loss.backward()
            opt.step()
            if lr_sched is not None:
                lr_sched.step()
            return loss.detach()

    # --train_dir: resume / checkpoint (rank-0-only writer, the reference examples' convention: tensorflow_mnist.py:159)
    ckpt = os.path.join(args.train_dir, "model.ckpt.pt") if args.train_dir else ""
    sched_step = 0   # the Horovod-API engine's schedule step count (the trainer keeps its own)
    if ckpt and os.path.exists(ckpt):
        sd = torch.load(ckpt, map_location="cpu", weights_only=False)
        # either engine reads what the other wrote: a trainer checkpoint carries masters / momentum / buffers by name, the
        # Horovod-API engine's a plain module state_dict + the optimizer's
        if args.b200_engine in ("fused", "nccl"):
            if "trainer" in sd:
                trainer.load_state_dict(sd["trainer"])
            else:
                names = {n for n, _ in model.named_parameters()}
                trainer.load_state_dict({"format": "b200mpi.DataParallelTrainer/1", "momentum": {},
                                         "model": {k: v for k, v in sd["model"].items() if k in names},
                                         "buffers": {k: v for k, v in sd["model"].items() if k not in names},
                                         "lr_schedule_step": sd.get("lr_schedule_step", 0)}, load_hyper=False)
        elif "trainer" in sd:
            model.load_state_dict({**sd["trainer"]["model"], **sd["trainer"]["buffers"]})
            sched_step = sd["trainer"].get("lr_schedule_step", 0)
        else:
            model.load_state_dict(sd["model"])
            opt.load_state_dict(sd["optimizer"])
            sched_step = sd.get("lr_schedule_step", 0)
        if rank == 0:
            print(f"Restored checkpoint from {ckpt} (written after {sd.get('batches', '?')} batches on {sd.get('world', '?')} ranks)")
            sys.stdout.flush()

    if lr_schedule is not None and args.b200_engine not in ("fused", "nccl"):
        for g in sgd.param_groups:   # the base rate, whatever rate the loaded optimizer state was at
            g["lr"] = g["initial_lr"] = lr
        lr_sched = torch.optim.lr_scheduler.LambdaLR(sgd, lambda e: lr_schedule.multiplier(sched_step + e))

    def save_checkpoint(batches_done):
        if not ckpt:
            return
        if args.b200_engine in ("fused", "nccl"):
            payload = {"trainer": trainer.state_dict()}          # collective: momentum shards are gathered
        else:
            payload = {"model": model.state_dict(), "optimizer": opt.state_dict()}
            if lr_sched is not None:
                payload["lr_schedule_step"] = sched_step + lr_sched.last_epoch
        if rank == 0:
            os.makedirs(args.train_dir, exist_ok=True)
            payload.update(batches=batches_done, world=size)
            torch.save(payload, ckpt + ".tmp")
            os.replace(ckpt + ".tmp", ckpt)
            print(f"Saved checkpoint to {ckpt}")
            sys.stdout.flush()

    def device_sync():
        if on_gpu:
            torch.cuda.synchronize()

    if evaluating:
        # forward-only pass over num_batches synthetic batches: tf_cnn_benchmarks' "Accuracy @ 1 = ... Accuracy @ 5 = ... [N examples]"
        if args.b200_engine not in ("fused", "nccl"):
            raise SystemExit("tf_cnn_benchmarks (b200): --eval needs the trainer engines (fused | nccl)")
        # with --moving_average_decay under the averaged weights, as tf_cnn_benchmarks' eval restores the averaged variables
        tot = {"top1": 0.0, "top5": 0.0, "n": 0}
        t_ev = time.perf_counter()
        with (trainer.ema_weights() if averaging else contextlib.nullcontext()):
            for _ in range(args.num_batches):
                r = trainer.evaluate(x, y)
                tot["top1"] += r.get("top1", 0.0)
                tot["top5"] += r.get("top5", 0.0)
                tot["n"] += r["examples"]
        device_sync()
        if rank == 0:
            print(f"Accuracy @ 1 = {tot['top1'] / args.num_batches:.4f} Accuracy @ 5 = {tot['top5'] / args.num_batches:.4f} [{tot['n']} examples]")
            print("----------------------------------------------------------------")
            print(f"total images/sec: {tot['n'] / (time.perf_counter() - t_ev):.2f}")
            print("----------------------------------------------------------------")
            sys.stdout.flush()
        hvd.shutdown()
        return

    for _ in range(args.num_warmup_batches):
        loss = step()
    device_sync()
    hvd.barrier()
    if rank == 0:
        print("Running warm up")
        print("Done warm up")
        print("Step\tImg/sec\ttotal_loss")
        sys.stdout.flush()
    speeds = []
    t_all = time.perf_counter()
    t0 = time.perf_counter()
    for i in range(1, args.num_batches + 1):
        loss = step()
        if i % args.display_every == 0 or i == 1:
            lv = float(loss)  # device->host read, syncs the step
            now = time.perf_counter()
            n = args.display_every if i > 1 else 1
            if i > 1:
                speeds.append(B * n / (now - t0))
            if rank == 0 and i > 1:
                import statistics
                cur = speeds[-1]
                unc = statistics.pstdev(speeds) / (len(speeds) ** 0.5) if len(speeds) > 1 else 0.0
                jitter = statistics.median([abs(s - statistics.median(speeds)) for s in speeds]) * 1.4826
                print(f"{i}\timages/sec: {cur:.1f} +/- {unc:.1f} (jitter = {jitter:.1f})\t{lv:.3f}")
                sys.stdout.flush()
            elif rank == 0:
                print(f"{i}\timages/sec: n/a (first step)\t{lv:.3f}")
            t0 = time.perf_counter()
    device_sync()
    hvd.barrier()
    total = args.num_batches * B * size / (time.perf_counter() - t_all)
    if rank == 0:
        print("----------------------------------------------------------------")
        print(f"total images/sec: {total:.2f}")
        print("----------------------------------------------------------------")
        sys.stdout.flush()
    save_checkpoint(args.num_warmup_batches + args.num_batches)
    hvd.shutdown()


if __name__ == "__main__":
    main()
