"""Parameter groups (per-group lr / momentum / weight decay) of DataParallelTrainer, on CPU.

The Communicator is an in-memory fake whose grouped fused allreduce+SGD does in PyTorch what the grouped
``k_allreduce_sgd`` does: every 4-element fp32 vector of the bucket takes ``{lr, momentum, weight_decay}`` from the row of
the group table that the bucket's slice of the group map names. The trainer is checked against
``torch.optim.SGD(param_groups)``; the kernel itself is covered by test_param_groups_gpu.py."""
import copy
import io

import pytest
import torch
import torch.nn as nn

from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer


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


class GroupComm:
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

    def allreduce_window(self, win, offset, count, dtype, op="sum", scale=None, algo=None, stream=None):
        self.launch_count += 1

    def allreduce_sgd_window(self, grad_win, grad_off, param_win, param_off, momentum, count, grad_dtype, lr,
                             momentum_coef=0.0, weight_decay=0.0, nesterov=False, first_step=False, scale=None,
                             lowp_win=None, lowp_off=0, algo=None, stream=None, group_map=None, group_hyper=None):
        self.launch_count += 1
        self.calls.append({"off": grad_off, "count": count, "grouped": group_map is not None})
        if group_map is not None:
            assert grad_dtype == torch.float32 and group_map.dtype == torch.uint8 and group_map.numel() == count // 4
            assert group_hyper.shape[1] == 3 and int(group_map.max()) < group_hyper.shape[0]
            h = group_hyper[group_map.long()]                       # [count / 4, 3]: each vector's row of the table
            lr, momentum_coef, weight_decay = h[:, 0:1], h[:, 1:2], h[:, 2:3]
        elif self.hyper is not None:
            lr, momentum_coef, weight_decay = (float(v) for v in self.hyper)
        g = grad_win.tensor(torch.float32, offset=grad_off, numel=count).view(-1, 4) * (1.0 if scale is None else scale)
        p = param_win.tensor(torch.float32, offset=param_off, numel=count).view(-1, 4)
        m = momentum[:count].view(-1, 4)
        g = g + weight_decay * p
        m.copy_(g if first_step else momentum_coef * m + g)
        p.sub_(lr * (g + momentum_coef * m if nesterov else m))
        if lowp_win is not None:
            lowp_win.tensor(torch.bfloat16, offset=lowp_off, numel=count).copy_(p.reshape(-1))


def small_cnn():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1, bias=False), nn.BatchNorm2d(8), nn.ReLU(),
                         nn.Conv2d(8, 16, 3, padding=1, bias=True), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(),
                         nn.Linear(16, 10))


def batches(n, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(4, 3, 8, 8, generator=g), torch.randint(0, 10, (4,), generator=g)) for _ in range(n)]


def recipe(model):
    """Three groups that interleave inside buckets: no decay on BN and biases, a faster classifier weight, the rest default."""
    no_wd = [p for n, p in model.named_parameters() if p.dim() == 1]
    head = [model[7].weight]
    return [{"params": no_wd, "weight_decay": 0.0}, {"params": head, "lr": 0.2, "momentum": 0.5}]


def reference(model, data, groups, lr, mu, wd, nesterov=False, autocast=False):
    listed = {id(p) for g in groups for p in g["params"]}
    rest = [p for p in model.parameters() if id(p) not in listed]
    opt = torch.optim.SGD([{"params": rest}] + groups, lr=lr, momentum=mu, weight_decay=wd, nesterov=nesterov)
    losses = []
    for x, y in data:
        opt.zero_grad()
        with torch.autocast("cpu", dtype=torch.bfloat16, enabled=autocast):
            loss = nn.CrossEntropyLoss()(model(x), y)
        loss.backward()
        losses.append(float(loss.detach()))
        opt.step()
    return losses


def trainer(model, groups, **kw):
    args = dict(lr=0.05, momentum=0.9, weight_decay=1e-3, bucket_bytes=1024, autocast_dtype=None, channels_last=False,
                cuda_graph=False)
    args.update(kw)
    return DataParallelTrainer(model, nn.CrossEntropyLoss(), GroupComm(), param_groups=groups, **args)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("nesterov", [False, True])
def test_groups_match_torch_sgd_across_buckets(fused, nesterov):
    ref = small_cnn()
    model = copy.deepcopy(ref)
    data = batches(4)
    want = reference(ref, data, recipe(ref), 0.05, 0.9, 1e-3, nesterov)
    tr = trainer(model, recipe(model), nesterov=nesterov, fused_optimizer=fused)
    assert len(tr.state.buckets) > 2
    got = [float(tr.step(x, y)) for x, y in data]
    assert got == pytest.approx(want, rel=1e-5)
    for a, b in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    if fused:
        assert tr.comm.calls and all(c["grouped"] for c in tr.comm.calls)


def test_groups_with_the_bf16_shadow_match_autocast_training():
    ref = small_cnn()
    model = copy.deepcopy(ref)
    data = batches(4)
    want = reference(ref, data, recipe(ref), 0.05, 0.9, 1e-3, autocast=True)
    tr = trainer(model, recipe(model), autocast_dtype=torch.bfloat16, bf16_params=True, bucket_bytes=2048)
    got = [float(tr.step(x, y)) for x, y in data]
    assert got == pytest.approx(want, rel=2e-3)
    for m, p, r in zip(tr.state.master_state().values(), model.parameters(), ref.parameters()):
        torch.testing.assert_close(m, r, rtol=2e-3, atol=2e-4)
        if p.dim() >= 2:
            assert torch.equal(p.detach(), m.to(torch.bfloat16))


@pytest.mark.parametrize("bf16", [False, True])
def test_group_map_marks_each_parameter_slot(bf16):
    model = small_cnn()
    tr = trainer(model, recipe(model), autocast_dtype=torch.bfloat16 if bf16 else None, bf16_params=bf16)
    st = tr.state
    gmap = st.group_map
    assert gmap.dtype == torch.uint8 and gmap.numel() == st.total // 4
    pad = 64 if bf16 else 4
    expect = torch.zeros_like(gmap)
    group_of = {id(p): 0 for p in model.parameters()}
    for k, g in enumerate(recipe(model), start=1):
        for p in g["params"]:
            group_of[id(p)] = k
    for p in model.parameters():
        start = st.param_slot[p][1]
        assert start % pad == 0
        n = (p.numel() + pad - 1) // pad * pad
        expect[start // 4:(start + n) // 4] = group_of[id(p)]
    assert torch.equal(gmap, expect)   # padding vectors follow their parameter; bucket tails stay group 0
    assert set(gmap.tolist()) == {0, 1, 2}
    for b in st.buckets:
        assert b.start % 8 == 0 and b.numel % 8 == 0
        assert torch.equal(st.bucket_group_map(b), gmap[b.start // 4:(b.start + b.numel) // 4])
    names = [g["params"] for g in tr.param_groups]
    assert names[2] == ["7.weight"] and set(names[1]) == {"1.weight", "1.bias", "3.bias", "7.bias"}
    assert set(names[0]) == {"0.weight", "3.weight"}


def test_set_lr_per_group_and_freezing():
    model = small_cnn()
    tr = trainer(model, recipe(model))
    tr.set_lr(0.0, group=2)
    assert [g["lr"] for g in tr.param_groups] == [0.05, 0.05, 0.0]
    assert tr.group_hyper[:, 0].tolist() == pytest.approx([0.05, 0.05, 0.0])
    head0 = model[7].weight.detach().clone()
    others0 = model[0].weight.detach().clone()
    for x, y in batches(2):
        tr.step(x, y)
    assert torch.equal(model[7].weight.detach(), head0)           # lr 0: bit-identical
    assert not torch.equal(model[0].weight.detach(), others0)
    tr.set_lr(0.01)
    assert [g["lr"] for g in tr.param_groups] == [0.01] * 3 and float(tr.hyper[0]) == pytest.approx(0.01)
    tr.set_lr(0.3, group=0)
    assert tr.param_groups[0]["lr"] == 0.3 and float(tr.hyper[0]) == pytest.approx(0.3)
    with pytest.raises(IndexError):
        tr.set_lr(0.1, group=3)


def test_no_groups_keeps_the_ungrouped_call():
    tr = trainer(small_cnn(), None)
    for x, y in batches(1):
        tr.step(x, y)
    assert tr.state.group_map is None and tr.group_hyper is None
    assert tr.comm.calls and not any(c["grouped"] for c in tr.comm.calls)
    assert [g["lr"] for g in tr.param_groups] == [0.05] and "param_groups" not in tr.state_dict()


@pytest.mark.parametrize("fused,bf16", [(True, False), (True, True), (False, False)])
def test_checkpoint_with_groups_continues_bit_for_bit(fused, bf16):
    data = batches(6, seed=4)
    kw = dict(fused_optimizer=fused, bf16_params=bf16, autocast_dtype=torch.bfloat16 if bf16 else None, bucket_bytes=2048)
    m = small_cnn()
    a = trainer(m, recipe(m), **kw)
    a.set_lr(0.02, group=1)
    for x, y in data[:3]:
        a.step(x, y)
    blob = io.BytesIO()
    torch.save(a.state_dict(), blob)
    for x, y in data[3:]:
        a.step(x, y)
    sd = torch.load(io.BytesIO(blob.getvalue()), weights_only=False)
    assert [g["lr"] for g in sd["param_groups"]] == [0.05, 0.02, 0.2]
    torch.manual_seed(99)
    fresh = small_cnn()
    with torch.no_grad():
        for p in fresh.parameters():
            p.add_(1.0)
    b = trainer(fresh, recipe(fresh), **dict(kw, lr=0.5))
    b.load_state_dict(sd)
    assert b.param_groups == a.param_groups
    for x, y in data[3:]:
        b.step(x, y)
    for (n, p), (_, q) in zip(a.state.master_state().items(), b.state.master_state().items()):
        assert torch.equal(p, q), n
    # load_hyper=False keeps this trainer's values
    mc = small_cnn()
    c = trainer(mc, recipe(mc), **dict(kw, lr=0.5))
    c.load_state_dict(sd, load_hyper=False)
    assert [g["lr"] for g in c.param_groups] == [0.5, 0.5, 0.2]


def test_checkpoint_group_mismatches_are_rejected():
    m = small_cnn()
    sd = trainer(m, recipe(m)).state_dict()
    plain = trainer(small_cnn(), None)
    with pytest.raises(ValueError, match="parameter groups"):
        plain.load_state_dict(sd)
    plain.load_state_dict(sd, load_hyper=False)
    m2 = small_cnn()
    with pytest.raises(ValueError, match="parameter groups"):
        trainer(m2, recipe(m2)).load_state_dict(plain.state_dict())
    m3 = small_cnn()
    other = trainer(m3, [{"params": [m3[7].weight, m3[7].bias], "lr": 0.2}, {"params": [m3[1].weight], "weight_decay": 0.0}])
    with pytest.raises(ValueError, match="other members"):
        other.load_state_dict(sd)
    old = {k: v for k, v in plain.state_dict().items()}
    trainer(small_cnn(), None).load_state_dict(old)        # no groups on either side: as before


def test_invalid_groups_raise_value_error():
    m = small_cnn()
    w = m[0].weight
    with pytest.raises(ValueError, match="twice"):
        trainer(m, [{"params": [w]}, {"params": [w]}])
    with pytest.raises(ValueError, match="twice"):
        trainer(m, [{"params": [w, w]}])
    with pytest.raises(ValueError, match="not a trainable parameter"):
        trainer(m, [{"params": [torch.zeros(3, requires_grad=True)]}])
    m[1].bias.requires_grad_(False)
    with pytest.raises(ValueError, match="not a trainable parameter"):
        trainer(m, [{"params": [m[1].bias]}])
    m = small_cnn()
    with pytest.raises(ValueError, match="unsupported keys"):
        trainer(m, [{"params": [m[0].weight], "dampening": 0.1}])
    with pytest.raises(ValueError, match="nesterov"):
        trainer(m, [{"params": [m[0].weight], "nesterov": True}])
    trainer(m, [{"params": [m[0].weight], "nesterov": False}])   # the trainer's own value is accepted
    with pytest.raises(ValueError, match="'params'"):
        trainer(m, [{"lr": 0.1}])
    with pytest.raises(ValueError, match="at most 255"):
        trainer(m, [{"params": []} for _ in range(256)])
    tr = trainer(m, [{"params": []} for _ in range(255)] + [])
    assert len(tr.param_groups) == 256 and tr.group_hyper.shape == (256, 3)
