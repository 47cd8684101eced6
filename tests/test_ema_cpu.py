"""DataParallelTrainer's weight average (``ema_decay``) on CPU.

A fake communicator does here, per rank thread, what the fused kernels do: the owner of each slice averages the ranks'
gradients, applies the SGD or LARS update to its fp32 slice, pushes the parameters (and the bf16 shadow) to every rank,
and folds them into its EMA shard with the exact oracle of tests/ema_oracle.py. The trainer's host logic around it (the
update count, ``no_sync``, ``ema_weights()``, checkpoints and re-sharding, the unfused path, the tf_cnn_benchmarks flag) is
checked against that oracle. The kernels themselves: test_ema_gpu.py."""
import copy
import os
import re
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch
import torch.nn as nn

from ema_oracle import ema_coef, ema_step
from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer

EPS = 1e-8


class Win:
    def __init__(self, wid, nbytes):
        self.id, self.nbytes = wid, nbytes
        self.buf = torch.zeros(nbytes, dtype=torch.uint8)

    def tensor(self, dtype=None, rank=-1, offset=0, numel=None):
        dtype = dtype or torch.uint8
        esz = torch.empty((), dtype=dtype).element_size()
        if numel is None:
            numel = (self.nbytes - offset) // esz
        return self.buf[offset:offset + numel * esz].view(dtype)


class World:
    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world)
        self.windows = {}
        self.shards = {}
        self.lock = threading.Lock()


class EmaComm:
    """One rank of a thread world (world 1 included)."""
    device = "cpu"

    def __init__(self, tw, rank=0):
        self.tw, self.rank, self.world = tw, rank, tw.world
        self.windows, self.launch_count, self.hyper, self.calls = [], 0, None, []

    def alloc_window(self, nbytes):
        w = Win(len(self.windows), nbytes)
        self.windows.append(w)
        with self.tw.lock:
            self.tw.windows.setdefault(w.id, {})[self.rank] = w
        return w

    def slice_elems(self, count, dtype):
        nvec = (count + 3) // 4
        return (nvec + self.world - 1) // self.world * 4

    def set_hyper(self, t):
        self.hyper = t

    def host_barrier(self):
        self.tw.barrier.wait(timeout=60)

    def lars_scratch_bytes(self, count, num_params):
        return 16

    def broadcast(self, tensor, root=0, stream=None):
        self.tw.barrier.wait(timeout=60)
        if self.rank != root:
            tensor.copy_(self.tw.windows[0][root].tensor(torch.float32)[:tensor.numel()])
        self.tw.barrier.wait(timeout=60)

    def allgather(self, shard, full):
        with self.tw.lock:
            self.tw.shards[self.rank] = shard.clone()
        self.tw.barrier.wait(timeout=60)
        full.copy_(torch.cat([self.tw.shards[r] for r in range(self.world)]))
        self.tw.barrier.wait(timeout=60)

    def allreduce_window(self, win, offset, count, dtype, op="sum", scale=None, algo=None, stream=None):
        self.launch_count += 1
        self.tw.barrier.wait(timeout=60)
        W = self.world
        g = sum(self.tw.windows[win.id][k].tensor(torch.float32, offset=offset, numel=count) for k in range(W)) / W
        self.tw.barrier.wait(timeout=60)
        win.tensor(torch.float32, offset=offset, numel=count).copy_(g)
        self.tw.barrier.wait(timeout=60)

    def _avg_grad(self, grad_win, grad_off, count, scale):
        W = self.world
        g = sum(self.tw.windows[grad_win.id][k].tensor(torch.float32, offset=grad_off, numel=count) for k in range(W))
        return g * (scale if scale is not None else 1.0 / W)

    def _finish(self, lo, hi, p_new, param_win, param_off, count, lowp_win, lowp_off, ema, ema_sched):
        for k in range(self.world):
            self.tw.windows[param_win.id][k].tensor(torch.float32, offset=param_off, numel=count)[lo:hi] = p_new
            if lowp_win is not None:
                self.tw.windows[lowp_win.id][k].tensor(torch.bfloat16, offset=lowp_off, numel=count)[lo:hi] = \
                    p_new.to(torch.bfloat16)
        if ema is not None:
            d, k = float(ema_sched[0]), int(ema_sched[1])
            ema[:hi - lo] = torch.from_numpy(ema_step(ema[:hi - lo].numpy(), p_new.numpy(), d, k))

    def allreduce_sgd_window(self, grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, lr,
                             momentum_coef=0.0, weight_decay=0.0, nesterov=False, first_step=False, scale=None,
                             lowp_win=None, lowp_off=0, algo=None, stream=None, **kw):
        self.launch_count += 1
        self.calls.append(("sgd", grad_off, count, lowp_off, sorted(kw)))
        r = self.rank
        per = self.slice_elems(count, torch.float32)
        lo, hi = min(r * per, count), min((r + 1) * per, count)
        self.tw.barrier.wait(timeout=60)
        if hi > lo:
            g = self._avg_grad(grad_win, grad_off, count, scale)[lo:hi]
            p = param_win.tensor(torch.float32, offset=param_off, numel=count)[lo:hi].clone()
            if kw.get("group_map") is not None:
                h = kw["group_hyper"][kw["group_map"].long()].repeat_interleave(4, 0)[lo:hi]
                lr_, mu, wd = h[:, 0], h[:, 1], h[:, 2]
            else:
                lr_, mu, wd = (float(v) for v in self.hyper)
            g = g + wd * p
            m = momentum[:hi - lo]
            m.copy_(g if first_step else mu * m + g)
            p = p - lr_ * (g + mu * m if nesterov else m)
            self._finish(lo, hi, p, param_win, param_off, count, lowp_win, lowp_off, kw.get("ema"), kw.get("ema_sched"))
        self.tw.barrier.wait(timeout=60)

    def allreduce_lars_window(self, grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, *, group_hyper,
                              param_map, param_table, board_win, board_off, scratch, trust_coefficient, nesterov=False,
                              first_step=False, scale=None, lowp_win=None, lowp_off=0, algo=None, stream=None,
                              trust_out=None, **kw):
        self.launch_count += 2
        self.calls.append(("lars", grad_off, count, lowp_off, sorted(kw)))
        r = self.rank
        per = self.slice_elems(count, torch.float32)
        lo, hi = min(r * per, count), min((r + 1) * per, count)
        self.tw.barrier.wait(timeout=60)
        g = self._avg_grad(grad_win, grad_off, count, scale).view(-1, 4)
        p = param_win.tensor(torch.float32, offset=param_off, numel=count).clone().view(-1, 4)
        P = param_table.shape[0]
        pid = param_map.long()
        gn = torch.zeros(P + 1).index_add_(0, pid, (g * g).sum(1))[:P].sqrt()
        wn = torch.zeros(P + 1).index_add_(0, pid, (p * p).sum(1))[:P].sqrt()
        grp, lars = param_table[:, 0].long(), param_table[:, 1].bool()
        wd_p = group_hyper[grp, 2]
        trust = torch.where(lars & (wn > 0) & (gn > 0), trust_coefficient * wn / (gn + wd_p * wn + EPS), torch.ones(P))
        if trust_out is not None:
            trust_out.copy_(trust)
        vt = torch.cat([trust, torch.ones(1)])[pid].repeat_interleave(4)
        vg = torch.cat([grp, torch.zeros(1, dtype=torch.long)])[pid].repeat_interleave(4)
        h = group_hyper[vg]
        g, p = g.reshape(-1), p.reshape(-1)
        self.tw.barrier.wait(timeout=60)                     # every rank has read the pre-update parameters
        if hi > lo:
            lr_, mu, wd = h[lo:hi, 0], h[lo:hi, 1], h[lo:hi, 2]
            d = vt[lo:hi] * (g[lo:hi] + wd * p[lo:hi])
            m = momentum[:hi - lo]
            m.copy_(d if first_step else mu * m + d)
            pn = p[lo:hi] - lr_ * (d + mu * m if nesterov else m)
            self._finish(lo, hi, pn, param_win, param_off, count, lowp_win, lowp_off, kw.get("ema"), kw.get("ema_sched"))
        self.tw.barrier.wait(timeout=60)


def small_cnn():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1, bias=False), nn.BatchNorm2d(8), nn.ReLU(),
                         nn.Conv2d(8, 16, 3, padding=1, bias=True), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(),
                         nn.Linear(16, 10))


def batches(n, bs=4, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(bs, 3, 8, 8, generator=g), torch.randint(0, 10, (bs,), generator=g)) for _ in range(n)]


def make(comm, model=None, **kw):
    kw = dict(dict(lr=0.1, momentum=0.9, weight_decay=1e-3, bucket_bytes=1024, autocast_dtype=None, channels_last=False,
                   cuda_graph=False), **kw)
    return DataParallelTrainer(model if model is not None else small_cnn(), nn.CrossEntropyLoss(), comm, **kw)


def run_world(world, fn):
    """fn(rank, comm) on `world` rank threads; returns {rank: result}."""
    tw = World(world)
    out, errs = {}, []

    def body(r):
        try:
            out[r] = fn(r, EmaComm(tw, r))
        except Exception as e:  # noqa: BLE001
            errs.append((r, repr(e)))
            tw.barrier.abort()
    ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    [t.start() for t in ts]
    [t.join(180) for t in ts]
    assert not errs and len(out) == world, errs
    return out


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def test_coefficient_schedule_is_the_oracle():
    assert float(ema_coef(0.9999, 1)) == float(np.float32(1 - 2 / 11))
    ks = [float(ema_coef(0.9999, k)) for k in range(1, 50)]
    assert ks == sorted(ks, reverse=True)
    assert float(ema_coef(0.999, 10 ** 6)) == float(np.float32(1 - float(np.float32(0.999))))


@pytest.mark.parametrize("lars", [False, True])
@pytest.mark.parametrize("groups", [False, True])
def test_fused_average_follows_the_parameters_and_no_sync(lars, groups):
    model = small_cnn()
    pg = [{"params": [p for p in model.parameters() if p.dim() == 1], "weight_decay": 0.0, "lars": False}] if groups else None
    tr = make(EmaComm(World(1)), model, ema_decay=0.99, lars=lars, param_groups=pg)
    st = tr.state
    e = st.flat_param.clone().numpy()                        # starts at the broadcast parameters
    assert tr.ema_updates == 0
    assert np.array_equal(tr._gather_ema().numpy().view(np.int32), e.view(np.int32))
    k = 0
    data = batches(6)
    for i, (x, y) in enumerate(data):
        if i in (2, 3):
            with tr.no_sync():                               # accumulation: no update, k does not move
                tr.step(x, y)
            assert tr.ema_updates == k
            assert np.array_equal(tr._gather_ema().numpy().view(np.int32), e.view(np.int32))
            continue
        tr.step(x, y)
        k += 1
        e = ema_step(e, st.flat_param.numpy(), 0.99, k)
        assert tr.ema_updates == k
        assert np.array_equal(tr._gather_ema().numpy().view(np.int32), e.view(np.int32))
    kinds = {c[0] for c in tr.comm.calls}
    assert kinds == ({"lars"} if lars else {"sgd"})
    assert all("ema" in c[4] and "ema_sched" in c[4] for c in tr.comm.calls)
    assert not np.any(tr._gather_ema().numpy()[st.flat_param.numpy() == 0] != 0)   # padding stays zero


@pytest.mark.parametrize("lars", [False, True])
def test_unfused_average_within_one_ulp_of_fused(lars):
    res = []
    for fused in (True, False):
        tr = make(EmaComm(World(1)), ema_decay=0.9, lars=lars, fused_optimizer=fused)
        for x, y in batches(5):
            tr.step(x, y)
        res.append((tr.state.flat_param.clone(), tr._gather_ema(), tr.ema_updates))
    assert res[0][2] == res[1][2] == 5
    torch.testing.assert_close(res[1][0], res[0][0], rtol=1e-5, atol=1e-6)
    # same update rule; the fused result is exact, the unfused one rounds the product separately
    tr = make(EmaComm(World(1)), ema_decay=0.9, fused_optimizer=False)
    e = tr.state.flat_param.clone().numpy()
    for k, (x, y) in enumerate(batches(5), 1):
        tr.step(x, y)
        want = ema_step(e, tr.state.flat_param.numpy(), 0.9, k)
        got = tr._gather_ema().numpy()
        ulp = np.spacing(np.abs(want)).astype(np.float32)
        assert np.all(np.abs(got.astype(np.float64) - want.astype(np.float64)) <= ulp), k
        e = want


@pytest.mark.parametrize("bf16", [False, True])
def test_ema_weights_swaps_in_and_restores_bit_for_bit(bf16):
    kw = dict(bf16_params=True, autocast_dtype=torch.bfloat16, bucket_bytes=2048) if bf16 else {}
    tr = make(EmaComm(World(1)), ema_decay=0.9, **kw)
    for x, y in batches(3):
        tr.step(x, y)
    st = tr.state
    p0 = st.flat_param.clone()
    l0 = None if st.flat_lowp is None else st.flat_lowp.clone()
    ema = tr._gather_ema()
    assert not torch.equal(ema, p0)
    x, y = batches(1, seed=7)[0]
    live = tr.evaluate(x, y)
    with tr.ema_weights():
        assert torch.equal(_bits(st.flat_param), _bits(ema))
        if bf16:
            assert torch.equal(st.flat_lowp, ema.to(torch.bfloat16))
            assert any(p.dtype == torch.bfloat16 for p in tr.model.parameters())
        averaged = tr.evaluate(x, y)
        with pytest.raises(RuntimeError, match="ema_weights"):
            tr.step(x, y)
        with pytest.raises(RuntimeError, match="ema_weights"):
            tr.state_dict()
        with pytest.raises(RuntimeError, match="already"):
            with tr.ema_weights():
                pass
    assert averaged["loss"] != live["loss"]
    assert torch.equal(_bits(st.flat_param), _bits(p0))
    if bf16:
        assert torch.equal(st.flat_lowp.view(torch.int16), l0.view(torch.int16))
    tr.step(x, y)                                            # training goes on from the restored parameters
    assert tr.ema_updates == 4


def test_ema_weights_needs_ema_decay():
    tr = make(EmaComm(World(1)))
    with pytest.raises(RuntimeError, match="ema_decay"):
        with tr.ema_weights():
            pass


@pytest.mark.parametrize("bad", [0, 0.0, 1, 1.0, -0.5, 1.5, float("nan"), float("inf"), True, "0.9"])
def test_bad_ema_decay_is_a_value_error(bad):
    with pytest.raises(ValueError, match="ema_decay"):
        make(EmaComm(World(1)), ema_decay=bad)


def test_without_ema_decay_nothing_changes():
    res = []
    for kw in ({}, {"ema_decay": None}):
        tr = make(EmaComm(World(1)), **kw)
        for x, y in batches(3):
            tr.step(x, y)
        res.append((tr.state_dict(), tr.comm.calls, tr.state.flat_param.clone()))
    (sd0, calls0, p0), (sd1, calls1, p1) = res
    assert set(sd0) == set(sd1) and "ema" not in sd1 and "ema_updates" not in sd1 and "ema_decay" not in sd1["hyper"]
    assert sd0["hyper"] == sd1["hyper"]
    assert calls0 == calls1 and all(c[4] == [] for c in calls1)       # the same calls, no EMA arguments
    assert torch.equal(p0, p1)


def _train_sd(world, steps, ema_decay=0.9, sd_in=None, bf16=False):
    data = batches(steps, bs=4 * world, seed=3)

    def fn(r, comm):
        kw = dict(bf16_params=True, autocast_dtype=torch.bfloat16, bucket_bytes=2048) if bf16 else {}
        tr = make(comm, ema_decay=ema_decay, **kw)
        if sd_in is not None:
            tr.load_state_dict(sd_in)
        for x, y in data:
            tr.step(x[4 * r:4 * r + 4], y[4 * r:4 * r + 4])
        return tr.state_dict()
    return run_world(world, fn)


def _assert_sd_equal(a, b):
    assert set(a) == set(b)
    for key in ("model", "momentum", "ema"):
        assert set(a[key]) == set(b[key])
        for n in a[key]:
            assert torch.equal(_bits(a[key][n]), _bits(b[key][n])), (key, n)
    assert a["ema_updates"] == b["ema_updates"] and a["hyper"] == b["hyper"]


def test_checkpoint_reshards_1_2_4_and_is_rank_independent():
    sd1 = _train_sd(1, 3)[0]
    assert sd1["ema_updates"] == 3 and sd1["hyper"]["ema_decay"] == float(np.float32(0.9))
    assert sd1["format"] == "b200mpi.DataParallelTrainer/1"
    for world in (2, 4):
        outs = _train_sd(world, 0, sd_in=sd1)                # load, no step, save: the same dictionary on every rank
        for r in range(world):
            _assert_sd_equal(outs[r], dict(sd1, world_size_at_save=world))
    # resume at world 2 from the world-1 checkpoint: every rank ends with the same average, k continues
    outs = _train_sd(2, 2, sd_in=sd1)
    _assert_sd_equal(outs[0], outs[1])
    assert outs[0]["ema_updates"] == 5


def test_multi_rank_average_is_identical_and_follows_the_parameters():
    data = batches(4, bs=8, seed=5)

    def fn(r, comm):
        tr = make(comm, ema_decay=0.95, bf16_params=True, autocast_dtype=torch.bfloat16, bucket_bytes=2048)
        e = tr.state.flat_param.clone().numpy()
        for k, (x, y) in enumerate(data, 1):
            tr.step(x[4 * r:4 * r + 4], y[4 * r:4 * r + 4])
            e = ema_step(e, tr.state.flat_param.numpy(), 0.95, k)
        with tr.ema_weights():
            inside = tr.state.flat_param.clone()
        return inside, e
    outs = run_world(2, fn)
    for r in range(2):
        assert torch.equal(_bits(outs[r][0]), _bits(outs[0][0]))
        assert np.array_equal(outs[r][0].numpy().view(np.int32), outs[r][1].view(np.int32))


def test_checkpoint_into_trainer_without_ema_and_the_reverse():
    sd = _train_sd(1, 2)[0]
    plain = make(EmaComm(World(1)))
    plain.load_state_dict(sd)                                # EMA keys ignored
    out = plain.state_dict()
    assert "ema" not in out and "ema_updates" not in out and "ema_decay" not in out["hyper"]
    for n in sd["model"]:
        assert torch.equal(out["model"][n], sd["model"][n])
    no_ema = _train_sd(1, 2, ema_decay=None)[0]
    assert "ema" not in no_ema
    tr = make(EmaComm(World(1)), ema_decay=0.99)
    tr.load_state_dict(no_ema)                               # the average restarts from the loaded masters, k = 0
    assert tr.ema_updates == 0
    assert torch.equal(tr._gather_ema(), tr.state.flat_param)
    tr2 = make(EmaComm(World(1)), ema_decay=0.99)            # a checkpoint with EMA: average and k come back
    tr2.load_state_dict(sd)
    assert tr2.ema_updates == 2 and tr2.ema_decay == float(np.float32(0.99))   # the decay stays this trainer's
    for n, v in tr2.state_dict()["ema"].items():
        assert torch.equal(v, sd["ema"][n])


def test_tf_cnn_benchmarks_moving_average_decay_trains_then_evaluates(tmp_path):
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    mpirun = os.path.join(repo, "mpi_operator_b200/bin/mpirun")
    if not os.path.exists(mpirun):
        pytest.skip("native launcher not built (run make)")
    script = os.path.join(repo, "examples/tensorflow-benchmarks/scripts/tf_cnn_benchmarks/tf_cnn_benchmarks.py")
    cmd = [mpirun, "-np", "2", sys.executable, script, "--device=cpu", "--model=trivial", "--batch_size=4", "--num_batches=3",
           "--num_warmup_batches=1", "--image_size=32", "--moving_average_decay=0.999", "--train_dir", str(tmp_path / "ckpt")]
    env = dict(os.environ, B200MPI_HVD_DEVICE="cpu")
    first = subprocess.run(cmd, capture_output=True, text=True, timeout=240, env=env, cwd="/tmp")
    assert first.returncode == 0 and "Saved checkpoint" in first.stdout, first.stdout[-1500:] + first.stderr[-2000:]
    assert "ignoring flags" not in first.stderr
    sd = torch.load(tmp_path / "ckpt" / "model.ckpt.pt", map_location="cpu", weights_only=False)["trainer"]
    assert sd["ema_updates"] == 4 and sd["hyper"]["ema_decay"] == float(np.float32(0.999))
    ev = subprocess.run(cmd + ["--eval=True"], capture_output=True, text=True, timeout=240, env=env, cwd="/tmp")
    assert ev.returncode == 0 and "Restored checkpoint" in ev.stdout, ev.stdout[-1500:] + ev.stderr[-2000:]
    m = re.search(r"Accuracy @ 1 = ([0-9.]+) Accuracy @ 5 = ([0-9.]+) \[(\d+) examples\]", ev.stdout)
    assert m and int(m.group(3)) == 3 * 4 * 2
