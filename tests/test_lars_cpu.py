"""LARS in DataParallelTrainer, on CPU.

The Communicator is an in-memory fake whose fused LARS step does in PyTorch what ``k_allreduce_lars_norms`` +
``k_lars_update`` do: per-parameter norms through the bucket's parameter map, the trust ratio, then the grouped SGD update
scaled by it. Both optimizer paths (that fake and ``fused_optimizer=False``) are checked against a float64 LARS written
here; the kernels themselves are covered by test_lars_gpu.py."""
import copy
import io

import pytest
import torch
import torch.nn as nn

from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer, FlatModelState

ETA = 0.02
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


class LarsComm:
    device = "cpu"
    rank, world = 0, 1

    def __init__(self):
        self.windows, self.launch_count, self.hyper, self.calls = [], 0, None, []

    def alloc_window(self, nbytes):
        self.windows.append(Win(len(self.windows), nbytes))
        return self.windows[-1]

    def slice_elems(self, count, dtype):
        return count

    def set_hyper(self, t):
        self.hyper = t

    def broadcast(self, tensor, root=0, stream=None):
        pass

    def host_barrier(self):
        pass

    def lars_scratch_bytes(self, count, num_params):
        return 16

    def allreduce_window(self, win, offset, count, dtype, op="sum", scale=None, algo=None, stream=None):
        self.launch_count += 1

    def allreduce_sgd_window(self, grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, lr,
                             momentum_coef=0.0, weight_decay=0.0, nesterov=False, first_step=False, scale=None,
                             lowp_win=None, lowp_off=0, algo=None, stream=None, group_map=None, group_hyper=None):
        self.launch_count += 1
        self.calls.append({"off": grad_off, "kind": "grouped" if group_map is not None else "sgd"})
        if group_map is not None:
            h = group_hyper[group_map.long()]
            lr, momentum_coef, weight_decay = h[:, 0:1], h[:, 1:2], h[:, 2:3]
        elif self.hyper is not None:
            lr, momentum_coef, weight_decay = (float(v) for v in self.hyper)
        self._update(grad_win, grad_off, param_win, param_off, momentum, count, scale, lr, momentum_coef, weight_decay,
                     1.0, nesterov, first_step, lowp_win, lowp_off)

    def allreduce_lars_window(self, grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, *, group_hyper,
                              param_map, param_table, board_win, board_off, scratch, trust_coefficient, nesterov=False,
                              first_step=False, scale=None, lowp_win=None, lowp_off=0, algo=None, stream=None,
                              trust_out=None):
        self.launch_count += 2
        self.calls.append({"off": grad_off, "kind": "lars"})
        P = param_table.shape[0]
        assert grad_dtype == torch.float32 and param_map.dtype == torch.uint16 and param_map.numel() == count // 4
        assert board_win.nbytes >= P * self.world * 8 and scratch.numel() >= self.lars_scratch_bytes(count, P)
        pid = param_map.long()
        assert bool((pid[1:] >= pid[:-1]).all()) and int(pid.max()) <= P
        g = grad_win.tensor(torch.float32, offset=grad_off, numel=count).view(-1, 4) * (1.0 if scale is None else scale)
        p = param_win.tensor(torch.float32, offset=param_off, numel=count).view(-1, 4)
        sg = torch.zeros(P + 1).index_add_(0, pid, (g * g).sum(1))[:P]
        sp = torch.zeros(P + 1).index_add_(0, pid, (p * p).sum(1))[:P]
        gn, wn = sg.sqrt(), sp.sqrt()
        grp, lars = param_table[:, 0].long(), param_table[:, 1].bool()
        wd_p = group_hyper[grp, 2]
        trust = torch.where(lars & (wn > 0) & (gn > 0), trust_coefficient * wn / (gn + wd_p * wn + EPS), torch.ones(P))
        if trust_out is not None:
            trust_out.copy_(trust)
        row = torch.cat([grp, grp.new_zeros(1)])[pid]
        h = group_hyper[row]
        self._update(grad_win, grad_off, param_win, param_off, momentum, count, scale, h[:, 0:1], h[:, 1:2], h[:, 2:3],
                     torch.cat([trust, trust.new_ones(1)])[pid].unsqueeze(1), nesterov, first_step, lowp_win, lowp_off)

    @staticmethod
    def _update(grad_win, grad_off, param_win, param_off, momentum, count, scale, lr, mu, wd, trust, nesterov, first_step,
                lowp_win, lowp_off):
        g = grad_win.tensor(torch.float32, offset=grad_off, numel=count).view(-1, 4) * (1.0 if scale is None else scale)
        p = param_win.tensor(torch.float32, offset=param_off, numel=count).view(-1, 4)
        m = momentum[:count].view(-1, 4)
        d = trust * (g + wd * p)
        m.copy_(d if first_step else mu * m + d)
        p.sub_(lr * (d + mu * m if nesterov else m))
        if lowp_win is not None:
            lowp_win.tensor(torch.bfloat16, offset=lowp_off, numel=count).copy_(p.reshape(-1))


class Net(nn.Module):
    """A BN CNN with a zero-initialised conv (|w| = 0 on the first step) and a layer forward never uses (|g| = 0)."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.conv1 = nn.Conv2d(3, 8, 3, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(8)
        self.conv2 = nn.Conv2d(8, 16, 3, padding=1, bias=True)
        self.fc = nn.Linear(16, 10)
        self.unused = nn.Linear(5, 3)
        nn.init.zeros_(self.conv2.weight)

    def forward(self, x):
        x = torch.relu(self.bn1(self.conv1(x)))
        x = torch.relu(self.conv2(x)).mean((2, 3))
        return self.fc(x)


def batches(n, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(4, 3, 8, 8, generator=g), torch.randint(0, 10, (4,), generator=g)) for _ in range(n)]


def recipe(model):
    """MLPerf's LARS recipe: BN and biases without LARS and weight decay; plus a head group with its own lr."""
    return [{"params": [p for p in model.parameters() if p.dim() == 1], "weight_decay": 0.0, "lars": False},
            {"params": [model.fc.weight], "lr": 0.2, "momentum": 0.5}]


def lars_reference(model, data, groups, lr, mu, wd, nesterov):
    """float64 LARS: returns the losses and the trust ratios of the last step by parameter name."""
    names = {id(p): n for n, p in model.named_parameters()}
    cfg = {n: (lr, mu, wd, True) for n in names.values()}
    for g in groups:
        for p in g["params"]:
            cfg[names[id(p)]] = (g.get("lr", lr), g.get("momentum", mu), g.get("weight_decay", wd), g.get("lars", True))
    model = copy.deepcopy(model).double()
    orig = dict(model.named_parameters())
    mom = {n: torch.zeros_like(p) for n, p in orig.items()}
    losses, trust = [], {}
    for x, y in data:
        model.zero_grad()
        loss = nn.CrossEntropyLoss()(model(x.double()), y)
        loss.backward()
        losses.append(float(loss.detach()))
        with torch.no_grad():
            for n, p in orig.items():
                l_, m_, w_, on = cfg[n]
                g = p.grad if p.grad is not None else torch.zeros_like(p)
                wn, gn = float(p.detach().norm()), float(g.norm())
                t = ETA * wn / (gn + w_ * wn + EPS) if (on and wn > 0 and gn > 0) else 1.0
                if on:
                    trust[n] = t
                d = t * (g + w_ * p)
                mom[n] = m_ * mom[n] + d
                p.sub_(l_ * (d + m_ * mom[n] if nesterov else mom[n]))
    return losses, dict(model.named_parameters()), trust


def make(model, groups, **kw):
    args = dict(lr=0.1, momentum=0.9, weight_decay=1e-3, bucket_bytes=1024, autocast_dtype=None, channels_last=False,
                cuda_graph=False, lars=True, trust_coefficient=ETA)
    args.update(kw)
    return DataParallelTrainer(model, nn.CrossEntropyLoss(), LarsComm(), param_groups=groups, **args)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("nesterov", [False, True])
def test_lars_matches_float64_reference(fused, nesterov):
    ref = Net()
    model = copy.deepcopy(ref)
    data = batches(4)
    want, ref_params, ref_trust = lars_reference(ref, data, recipe(ref), 0.1, 0.9, 1e-3, nesterov)
    tr = make(model, recipe(model), nesterov=nesterov, fused_optimizer=fused)
    assert len(tr.state.buckets) > 2
    got = [float(tr.step(x, y)) for x, y in data]
    assert got == pytest.approx(want, rel=1e-5)
    for n, p in model.named_parameters():
        torch.testing.assert_close(p.double(), ref_params[n].detach(), rtol=1e-5, atol=1e-6, msg=n)
    trust = tr.lars_trust_ratios()
    assert set(trust) == set(ref_trust) and "bn1.weight" not in trust and "conv1.weight" in trust
    for n, t in trust.items():
        assert t == pytest.approx(ref_trust[n], rel=1e-5), n
    assert trust["unused.weight"] == 1.0                     # no gradient: trust 1
    if fused:
        kinds = {c["kind"] for c in tr.comm.calls}
        assert "lars" in kinds


def test_zero_weight_gets_trust_one_on_its_first_step():
    model = Net()
    tr = make(model, recipe(model))
    x, y = batches(1)[0]
    tr.step(x, y)
    assert tr.lars_trust_ratios()["conv2.weight"] == 1.0
    tr.step(x, y)
    assert tr.lars_trust_ratios()["conv2.weight"] != 1.0


def test_lars_without_groups_builds_one_group_table():
    model = Net()
    tr = make(model, None)
    assert tr.group_hyper.shape == (1, 3) and tr.param_groups[0]["lars"] is True
    assert all(b.lars for b in tr.state.buckets)
    x, y = batches(1)[0]
    tr.set_lr(0.05)
    assert float(tr.group_hyper[0, 0]) == pytest.approx(0.05)
    tr.step(x, y)
    assert all(c["kind"] == "lars" for c in tr.comm.calls)


def test_default_off_keeps_todays_calls():
    m = Net()
    tr = make(m, recipe(m), lars=False)
    x, y = batches(1)[0]
    tr.step(x, y)
    assert tr.state.param_map is None and not any(b.lars for b in tr.state.buckets)
    assert tr.comm.calls and all(c["kind"] == "grouped" for c in tr.comm.calls)
    assert tr.lars_trust_ratios() == {}
    tr2 = make(Net(), None, lars=False)
    tr2.step(x, y)
    assert tr2.group_hyper is None and all(c["kind"] == "sgd" for c in tr2.comm.calls)


def test_buckets_without_lars_parameters_keep_the_grouped_kernel():
    m = Net()
    only_fc = [{"params": [p for n, p in m.named_parameters() if n != "fc.weight"], "lars": False}]
    tr = make(m, only_fc, bucket_bytes=256)
    x, y = batches(1)[0]
    tr.step(x, y)
    lars_buckets = [b for b in tr.state.buckets if b.lars]
    assert len(lars_buckets) == 1 and m.fc.weight in lars_buckets[0].params
    kinds = [c["kind"] for c in tr.comm.calls]
    assert kinds.count("lars") == 1 and kinds.count("grouped") == len(tr.state.buckets) - 1
    assert list(tr.lars_trust_ratios()) == ["fc.weight"]


@pytest.mark.parametrize("bf16", [False, True])
def test_parameter_map_marks_each_parameter_slot(bf16):
    m = Net()
    tr = make(m, recipe(m), bf16_params=bf16, autocast_dtype=torch.bfloat16 if bf16 else None)
    st = tr.state
    pmap = st.param_map.long()
    assert st.param_map.dtype == torch.uint16 and pmap.numel() == st.total // 4
    pad = 64 if bf16 else 4
    for b in st.buckets:
        local = pmap[b.start // 4:(b.start + b.numel) // 4]
        assert bool((local[1:] >= local[:-1]).all())
        covered = torch.zeros_like(local, dtype=torch.bool)
        for k, p in enumerate(b.params):
            start = st.param_slot[p][1]
            lo, hi = (start - b.start) // 4, (start - b.start + -(-p.numel() // pad) * pad) // 4
            assert bool((local[lo:hi] == k).all())                       # the parameter and its padding
            covered[lo:hi] = True
        assert bool((local[~covered] == len(b.params)).all())          # bucket tail: the dummy entry
        tab = b.param_table
        assert tab.shape == (len(b.params), 2)
        for k, p in enumerate(b.params):
            want_group = 1 if p.dim() == 1 else (2 if p is m.fc.weight else 0)
            assert int(tab[k, 0]) == want_group and bool(tab[k, 1]) == (p.dim() != 1)


def test_invalid_lars_arguments_raise_value_error():
    m = Net()
    with pytest.raises(ValueError, match="lars must be a bool"):
        make(m, None, lars=1)
    for eta in (0.0, -1.0, float("inf"), "0.1"):
        with pytest.raises(ValueError, match="trust_coefficient"):
            make(Net(), None, trust_coefficient=eta)
    m = Net()
    with pytest.raises(ValueError, match="'lars' must be a bool"):
        make(m, [{"params": [m.fc.weight], "lars": "yes"}])


def test_too_many_parameters_in_a_lars_bucket_is_a_value_error():
    class Wide(nn.Module):
        def __init__(self):
            super().__init__()
            self.ps = nn.ParameterList([nn.Parameter(torch.randn(2)) for _ in range(1030)])

    with pytest.raises(ValueError, match="bucket_bytes"):
        make(Wide(), None, bucket_bytes=1 << 20)
    make(Wide(), None, bucket_bytes=1 << 20, lars=False)       # SGD has no such cap
    make(Wide(), None, bucket_bytes=4096)                      # smaller buckets fit


def test_no_sync_accumulation_then_one_lars_step():
    """Two accumulated batches, one LARS step: the trust ratios are those of the summed gradient (float64 reference)."""
    data = batches(2, seed=5)
    model = Net()
    tr = make(model, recipe(model))
    with tr.no_sync():
        tr.step(*data[0])
    assert all(v == 1.0 for v in tr.lars_trust_ratios().values())     # nothing synchronised yet
    tr.step(*data[1])
    got = tr.lars_trust_ratios()
    ref = Net().double()
    for x, y in data:
        nn.CrossEntropyLoss()(ref(x.double()), y).backward()
    for n, p in ref.named_parameters():
        if p.dim() == 1:
            continue
        g = p.grad if p.grad is not None else torch.zeros_like(p)
        wn, gn = float(p.norm()), float(g.norm())
        want = ETA * wn / (gn + 1e-3 * wn + EPS) if (wn > 0 and gn > 0) else 1.0
        assert got[n] == pytest.approx(want, rel=1e-5), n


@pytest.mark.parametrize("fused", [True, False])
def test_checkpoint_with_lars_continues_bit_for_bit(fused):
    data = batches(6, seed=4)
    kw = dict(fused_optimizer=fused, bucket_bytes=2048)
    m = Net()
    a = make(m, recipe(m), **kw)
    for x, y in data[:3]:
        a.step(x, y)
    blob = io.BytesIO()
    torch.save(a.state_dict(), blob)
    for x, y in data[3:]:
        a.step(x, y)
    sd = torch.load(io.BytesIO(blob.getvalue()), weights_only=False)
    assert [g["lars"] for g in sd["param_groups"]] == [True, False, True]
    assert sd["hyper"]["trust_coefficient"] == ETA and sd["hyper"]["lars"] is True
    fresh = Net()
    with torch.no_grad():
        for p in fresh.parameters():
            p.add_(1.0)
    b = make(fresh, recipe(fresh), **dict(kw, lr=0.5))
    b.load_state_dict(sd)
    assert b.param_groups == a.param_groups
    for x, y in data[3:]:
        b.step(x, y)
    for (n, p), (_, q) in zip(a.state.master_state().items(), b.state.master_state().items()):
        assert torch.equal(p, q), n
    assert a.lars_trust_ratios() == b.lars_trust_ratios()


def test_sgd_and_lars_checkpoints_load_into_each_other():
    data = batches(3, seed=2)
    m = Net()
    sgd = make(m, recipe(m), lars=False)
    for x, y in data:
        sgd.step(x, y)
    sd = sgd.state_dict()
    m2 = Net()
    lars = make(m2, recipe(m2))
    lars.load_state_dict(sd)
    assert [g["lars"] for g in lars.param_groups] == [True, False, True]      # built with LARS, stays LARS
    for (n, p), (_, q) in zip(sgd.state.master_state().items(), lars.state.master_state().items()):
        assert torch.equal(p, q), n
    assert torch.equal(torch.cat([b.momentum for b in sgd.state.buckets]), torch.cat([b.momentum for b in lars.state.buckets]))
    m3 = Net()
    back = make(m3, recipe(m3), lars=False)
    back.load_state_dict(lars.state_dict())
    assert not any(g["lars"] for g in back.param_groups)
    for (n, p), (_, q) in zip(back.state.master_state().items(), lars.state.master_state().items()):
        assert torch.equal(p, q), n
    # a checkpoint without groups (plain SGD) into a LARS trainer without groups
    plain = make(Net(), None, lars=False)
    plain.step(*data[0])
    nog = make(Net(), None)
    nog.load_state_dict(plain.state_dict())
    assert float(nog.group_hyper[0, 0]) == pytest.approx(0.1)


def test_flat_state_builds_no_map_without_lars():
    st = FlatModelState(Net(), LarsComm(), 1024)
    assert st.param_map is None and not any(b.lars for b in st.buckets)
