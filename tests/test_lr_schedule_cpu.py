"""Learning-rate schedules (``LRSchedule``, ``DataParallelTrainer(lr_schedule=...)``) on CPU, against the exact oracle of
tests/lr_schedule_oracle.py.

The trainer runs on the thread-per-rank fake communicator of test_ema_cpu.py, whose fused SGD / LARS calls read the
learning rate from the trainer's tables as the kernels do; on a CPU device the trainer writes those tables from
``LRSchedule.rate``. The kernel itself: test_lr_schedule_gpu.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import lr_schedule_oracle as O
from mpi_operator_b200.parallel.lr_schedule import LRSchedule
from test_ema_cpu import EmaComm, World, batches, make, run_world, small_cnn
from test_lr_schedule_oracle_cpu import BASES, SPECS


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


@pytest.mark.parametrize("spec", SPECS, ids=[f"{s['form']}-W{s['warmup_steps']}" for s in SPECS])
def test_schedule_is_the_oracle_bit_for_bit(spec):
    sch = LRSchedule.from_dict(spec)
    assert sch.to_dict() == spec and LRSchedule.from_dict(sch.to_dict()) == sch
    for k in O.k_grid(spec):
        m = O.multiplier(spec, k)
        assert np.float64(sch.multiplier(k)).view(np.int64) == np.float64(m).view(np.int64), k
        for base in BASES + O.edge_bases(m):
            assert np.float32(sch.rate(base, k)).view(np.int32) == O.rate(spec, base, k).view(np.int32), (k, base)


def test_constructors():
    assert LRSchedule.constant().to_dict() == {"form": "constant", "warmup_steps": 0}
    assert LRSchedule.piecewise([5], [1, 0.1], warmup_steps=2).multiplier(1) == 0.5
    assert LRSchedule.exponential(10, 0.5).multiplier(25) == 0.25
    p = LRSchedule.polynomial(100, warmup_steps=10)
    assert p.power == 2 and p.end == 0.0 and p.multiplier(10) == 1.0 and p.multiplier(100) == 0.0
    assert p.table() == [10.0, 100.0, 2.0, 0.0]
    assert LRSchedule.piecewise([3, 7], [1.0, 0.5, 0.25]).table() == [0.0, 3.0, 7.0, 1.0, 0.5, 0.25]


@pytest.mark.parametrize("build, match", [
    (lambda: LRSchedule.piecewise([1, 2], [1.0, float("nan"), 0.5]), "multipliers"),
    (lambda: LRSchedule.piecewise([1, 2], [1.0, float("inf"), 0.5]), "multipliers"),
    (lambda: LRSchedule.piecewise([1, 2], [1.0, -0.1, 0.5]), "multipliers"),
    (lambda: LRSchedule.exponential(10, -0.5), "factor"),
    (lambda: LRSchedule.exponential(10, float("nan")), "factor"),
    (lambda: LRSchedule.exponential(10, 0.5, floor=-1.0), "floor"),
    (lambda: LRSchedule.exponential(10, 0.5, floor=float("inf")), "floor"),
    (lambda: LRSchedule.polynomial(10, end=-0.1), "end"),
    (lambda: LRSchedule.polynomial(10, end=float("nan")), "end"),
    (lambda: LRSchedule.constant(warmup_steps=-1), "warmup_steps"),
    (lambda: LRSchedule.constant(warmup_steps=2.5), "warmup_steps"),
    (lambda: LRSchedule.constant(warmup_steps=True), "warmup_steps"),
    (lambda: LRSchedule.piecewise([3, 2], [1.0, 0.5, 0.25]), "increasing"),
    (lambda: LRSchedule.piecewise([2, 2], [1.0, 0.5, 0.25]), "increasing"),
    (lambda: LRSchedule.piecewise([-1], [1.0, 0.5]), "boundaries"),
    (lambda: LRSchedule.piecewise(list(range(65)), [1.0] * 66), "at most 64"),
    (lambda: LRSchedule.piecewise([1, 2], [1.0, 0.5]), "multipliers"),
    (lambda: LRSchedule.piecewise([1], [1.0, 0.5, 0.1]), "multipliers"),
    (lambda: LRSchedule.exponential(0, 0.5), "decay_steps"),
    (lambda: LRSchedule.polynomial(10, warmup_steps=10), "total_steps"),
    (lambda: LRSchedule.polynomial(10, warmup_steps=11), "total_steps"),
    (lambda: LRSchedule.polynomial(10, power=0), "power"),
    (lambda: LRSchedule.polynomial(10, power=65), "power"),
    (lambda: LRSchedule.polynomial(10, power=1.5), "power"),
    (lambda: LRSchedule.from_dict({"form": "cosine"}), "LRSchedule"),
])
def test_validation_errors(build, match):
    with pytest.raises(ValueError, match=match):
        build()


def test_trainer_rejects_a_non_schedule():
    with pytest.raises(ValueError, match="lr_schedule"):
        make(EmaComm(World(1)), lr_schedule=lambda k: 1.0)


def _groups(model, on):
    return [{"params": [p for p in model.parameters() if p.dim() == 1], "weight_decay": 0.0, "lr": 0.37, "lars": False}] \
        if on else None


SCHED = {"form": "piecewise", "warmup_steps": 3, "boundaries": [4, 6], "multipliers": [1.0, 0.1, 0.01]}


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("kind", ["sgd", "groups", "lars"])
def test_trainer_tables_follow_the_oracle_every_step(world, kind):
    data = batches(8, bs=4 * world, seed=11)
    models = [small_cnn() for _ in range(world)]   # small_cnn seeds the global generator: not inside the rank threads

    def fn(r, comm):
        model = models[r]
        tr = make(comm, model, lr=0.1, lars=kind == "lars", param_groups=_groups(model, kind == "groups"),
                  lr_schedule=LRSchedule.from_dict(SCHED))
        bases = [g["lr"] for g in tr.param_groups]
        fixed = tr.group_hyper[:, 1:].clone() if tr.group_hyper is not None else None
        seen = []
        for k, (x, y) in enumerate(data):
            tr.step(x[4 * r:4 * r + 4], y[4 * r:4 * r + 4])
            want = [O.rate(SCHED, b, k) for b in bases]
            got = np.array(tr.current_lrs(), dtype=np.float32)
            assert np.array_equal(got.view(np.int32), np.array(want, dtype=np.float32).view(np.int32)), (k, got, want)
            assert np.float32(float(tr.hyper[0])).view(np.int32) == want[0].view(np.int32)
            if fixed is not None:
                assert torch.equal(tr.group_hyper[:, 1:], fixed)      # momentum and weight decay untouched
            assert tr.lr_schedule_step == k + 1
            seen.append(tr.state.flat_param.clone())
        assert [g["lr"] for g in tr.param_groups] == bases              # base rates reported
        return seen
    outs = run_world(world, fn)
    for r in range(world):                                              # every rank holds the same parameters
        for a, b in zip(outs[r], outs[0]):
            assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("kind", ["sgd", "groups", "lars"])
@pytest.mark.parametrize("fused", [True, False])
def test_equivalent_to_set_lr_before_each_step(kind, fused):
    data = batches(7, seed=4)
    res = []
    for scheduled in (True, False):
        model = small_cnn()
        tr = make(EmaComm(World(1)), model, lr=0.1, lars=kind == "lars", param_groups=_groups(model, kind == "groups"),
                  fused_optimizer=fused, lr_schedule=LRSchedule.from_dict(SCHED) if scheduled else None)
        bases = [g["lr"] for g in tr.param_groups]
        for k, (x, y) in enumerate(data):
            if not scheduled:
                for g, b in enumerate(bases):
                    tr.set_lr(float(O.rate(SCHED, b, k)), group=g)
            tr.step(x, y)
        mom = tr._gather_shards("momentum") if fused else tr._flat_mom
        res.append((tr.state.flat_param.clone(), mom.clone()))
    assert torch.equal(_bits(res[0][0]), _bits(res[1][0])) and torch.equal(_bits(res[0][1]), _bits(res[1][1]))


def test_first_step_sets_the_momentum_but_moves_no_parameter():
    tr = make(EmaComm(World(1)), lr_schedule=LRSchedule.constant(warmup_steps=4))
    p0 = tr.state.flat_param.clone()
    tr.step(*batches(1)[0])
    assert tr.current_lrs() == [0.0]
    assert torch.equal(_bits(tr.state.flat_param), _bits(p0))
    assert tr._gather_shards("momentum").abs().sum() > 0


def test_no_sync_does_not_advance_k():
    tr = make(EmaComm(World(1)), lr_schedule=LRSchedule.from_dict(SCHED))
    data = batches(5)
    tr.step(*data[0])
    with tr.no_sync():
        tr.step(*data[1])
        tr.step(*data[2])
    assert tr.lr_schedule_step == 1
    tr.step(*data[3])
    assert tr.lr_schedule_step == 2 and tr.current_lrs() == [float(O.rate(SCHED, 0.1, 1))]


def test_set_lr_rescales_the_base():
    model = small_cnn()
    tr = make(EmaComm(World(1)), model, lr=0.1, param_groups=_groups(model, True), lr_schedule=LRSchedule.from_dict(SCHED))
    data = batches(6)
    for x, y in data[:4]:
        tr.step(x, y)
    tr.set_lr(0.5, group=1)
    assert [g["lr"] for g in tr.param_groups] == [0.1, 0.5]
    assert tr.current_lrs() == [float(O.rate(SCHED, 0.1, 3)), float(O.rate(SCHED, 0.37, 3))]   # until the next step
    tr.step(*data[4])
    assert tr.current_lrs() == [float(O.rate(SCHED, 0.1, 4)), float(O.rate(SCHED, 0.5, 4))]
    tr.set_lr(2.0)
    tr.step(*data[5])
    assert tr.current_lrs() == [float(O.rate(SCHED, 2.0, 5))] * 2
    assert tr.state_dict()["hyper"]["lr"] == 2.0


def _run(steps, sd_in=None, world=1, **kw):
    data = batches(8, bs=4 * world, seed=9)
    models = [small_cnn() for _ in range(world)]   # small_cnn seeds the global generator: not inside the rank threads

    def fn(r, comm):
        model = models[r]
        tr = make(comm, model, lr_schedule=LRSchedule.from_dict(SCHED), param_groups=_groups(model, True), **kw)
        if sd_in is not None:
            tr.load_state_dict(sd_in)
        k0 = tr.lr_schedule_step
        for x, y in data[k0:k0 + steps]:
            tr.step(x[4 * r:4 * r + 4], y[4 * r:4 * r + 4])
        return tr, tr.state_dict()
    return run_world(world, fn)


@pytest.mark.parametrize("world", [1, 2])
def test_checkpoint_round_trip_continues_bit_for_bit(world):
    straight = _run(7, world=world)[0]
    half = _run(3, world=world)[0][1]
    assert half["lr_schedule_step"] == 3 and half["lr_schedule"] == SCHED
    assert [g["lr"] for g in half["param_groups"]] == [0.1, 0.37] and half["hyper"]["lr"] == 0.1
    tr, sd = _run(4, sd_in=half, world=world)[0]
    assert sd["lr_schedule_step"] == 7
    assert tr.current_lrs() == straight[0].current_lrs()
    for key in ("model", "momentum"):
        for n in sd[key]:
            assert torch.equal(_bits(sd[key][n]), _bits(straight[1][key][n])), (key, n)
    # loading restores k and what the last step used; the trainer keeps its own schedule
    other = make(EmaComm(World(1)), lr_schedule=LRSchedule.constant())
    other.load_state_dict(half, load_hyper=False)
    assert other.lr_schedule_step == 3 and other.lr_schedule == LRSchedule.constant()


def test_checkpoint_without_schedule_keys_starts_at_zero_and_plain_trainer_ignores_them():
    plain_sd = make(EmaComm(World(1))).state_dict()
    tr = make(EmaComm(World(1)), lr_schedule=LRSchedule.from_dict(SCHED))
    tr.step(*batches(1)[0])
    tr.load_state_dict(plain_sd)
    assert tr.lr_schedule_step == 0
    sd = _run(2)[0][1]
    model = small_cnn()
    plain = make(EmaComm(World(1)), model, param_groups=_groups(model, True))
    plain.load_state_dict(sd)
    out = plain.state_dict()
    assert "lr_schedule" not in out and "lr_schedule_step" not in out
    assert plain.current_lrs() == [float(np.float32(0.1)), float(np.float32(0.37))]


def test_without_schedule_nothing_changes():
    res = []
    for kw in ({}, {"lr_schedule": None}, {"lr_schedule": LRSchedule.constant()}):
        tr = make(EmaComm(World(1)), **kw)
        for x, y in batches(3):
            tr.step(x, y)
        res.append((tr.state_dict(), tr.comm.calls, tr.state.flat_param.clone(), tr.comm.launch_count))
    (sd0, calls0, p0, n0), (sd1, calls1, p1, n1), (sd2, _, p2, _) = res
    assert set(sd0) == set(sd1) and "lr_schedule" not in sd1 and "lr_schedule_step" not in sd1
    assert sd0["hyper"] == sd1["hyper"] and calls0 == calls1 and n0 == n1
    for key in ("model", "momentum"):
        for n in sd0[key]:
            assert torch.equal(sd0[key][n], sd1[key][n])
    # a constant schedule without warm-up trains exactly like no schedule
    assert torch.equal(_bits(p0), _bits(p1)) and torch.equal(_bits(p0), _bits(p2))
    assert set(sd2) == set(sd0) | {"lr_schedule", "lr_schedule_step"}


def _script(tmp_path, *flags, np_=2, ckpt="ckpt"):
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    mpirun = os.path.join(repo, "mpi_operator_b200/bin/mpirun")
    if not os.path.exists(mpirun):
        pytest.skip("native launcher not built (run make)")
    script = os.path.join(repo, "examples/tensorflow-benchmarks/scripts/tf_cnn_benchmarks/tf_cnn_benchmarks.py")
    cmd = [mpirun, "-np", str(np_), sys.executable, script, "--device=cpu", "--model=trivial", "--batch_size=4",
           "--num_batches=3", "--num_warmup_batches=1", "--image_size=32", "--train_dir", str(tmp_path / ckpt), *flags]
    env = dict(os.environ, B200MPI_HVD_DEVICE="cpu")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=240, env=env, cwd="/tmp")
    assert out.returncode == 0 and "Saved checkpoint" in out.stdout, out.stdout[-1500:] + out.stderr[-2000:]
    assert "ignoring flags" not in out.stderr
    return out, torch.load(tmp_path / ckpt / "model.ckpt.pt", map_location="cpu", weights_only=False)


# 1281167 / (4 x 2) images per step: 160145.875 steps per epoch
SPE = 1281167.0 / 8


def test_tf_cnn_benchmarks_schedule_flags_on_the_hvd_engine_and_resume(tmp_path):
    flags = ("--init_learning_rate=0.05", "--num_learning_rate_warmup_epochs=0.00002", "--num_epochs_per_decay=0.00001",
             "--learning_rate_decay_factor=0.5", "--minimum_learning_rate=0.01")
    out, sd = _script(tmp_path, *flags)
    want = LRSchedule.exponential(int(SPE * 0.00001), 0.5, floor=0.01 / 0.05, warmup_steps=int(SPE * 0.00002))
    assert f"x {want!r}" in out.stdout and "LR:          0.1 " in out.stdout
    assert sd["lr_schedule_step"] == 4
    _, sd = _script(tmp_path, *flags)                                      # resumes from the checkpoint: k continues
    assert sd["lr_schedule_step"] == 8


def test_tf_cnn_benchmarks_piecewise_on_the_trainer_and_resume(tmp_path):
    # --moving_average_decay makes the host run use the trainer (unfused optimizer), whose tables follow the schedule
    flags = ("--piecewise_learning_rate_schedule=0.2;0.00001;0.02;0.00003;0.002", "--num_learning_rate_warmup_epochs=0.00001",
             "--moving_average_decay=0.9")
    out, sd = _script(tmp_path, *flags)
    want = LRSchedule.piecewise([int(SPE * 0.00001), int(SPE * 0.00003)], [1.0, 0.1, 0.01], warmup_steps=int(SPE * 0.00001))
    tsd = sd["trainer"]
    assert LRSchedule.from_dict(tsd["lr_schedule"]).boundaries == want.boundaries == [1, 4]
    assert tsd["lr_schedule_step"] == 4 and tsd["hyper"]["lr"] == 0.4               # base: v0 x world
    _, sd = _script(tmp_path, *flags)
    assert sd["trainer"]["lr_schedule_step"] == 8


def test_tf_cnn_benchmarks_rejects_a_bad_schedule(tmp_path):
    with pytest.raises(AssertionError, match="learning-rate schedule"):
        _script(tmp_path, "--piecewise_learning_rate_schedule=0.1;1", np_=1)
