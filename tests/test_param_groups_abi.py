"""CPU-side checks of parameter groups in FlatAdam / ShardedFlatAdam: group validation, the segment table, the
state_dict format against torch.optim.Adam / AdamW built on CPU with the same groups, and C2V_EINVAL from the grouped
entry points before any CUDA call.  Nothing here launches a kernel."""
import ctypes
import io

import pytest
import torch
import torch.nn as nn
from torch.optim import lr_scheduler as LS

from code2vec_b200 import _lib
from code2vec_b200.distributed import FlatAdam, FlatGradBucket, ShardedFlatAdam

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
ODD = V(0x1004)


class Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(11, 6)
        self.path = nn.Embedding(7, 5)
        self.lin = nn.Linear(6, 3)
        self.norm = nn.LayerNorm(3)


def _recipe(net, wd=0.01):
    decay = [net.emb.weight, net.path.weight, net.lin.weight]
    return [{"params": decay, "weight_decay": wd}, {"params": [net.lin.bias, net.norm.weight, net.norm.bias],
                                                    "weight_decay": 0.0, "lr": 5e-4}]


def _make(kind, net, groups, **kw):
    if kind == "flat":
        return FlatAdam(FlatGradBucket(net.parameters()), groups=groups, **kw)
    if kind == "sharded":
        return ShardedFlatAdam(groups, **kw)
    return ShardedFlatAdam(groups, early=[net.path.weight], **kw)


KINDS = ["flat", "sharded", "sharded-early"]


@pytest.mark.parametrize("kind", KINDS)
def test_groups_take_the_constructors_defaults(kind):
    net = Net()
    opt = _make(kind, net, _recipe(net), lr=1e-3, betas=(0.8, 0.99), decoupled_weight_decay=True, max_grad_norm=1.0)
    g0, g1 = opt.param_groups
    assert (g0["lr"], g1["lr"], g0["weight_decay"], g1["weight_decay"]) == (1e-3, 5e-4, 0.01, 0.0)
    assert g0["betas"] == g1["betas"] == (0.8, 0.99) and g0["decoupled_weight_decay"] and g1["decoupled_weight_decay"]
    assert opt.max_grad_norm == 1.0
    for name in ("lr", "betas", "eps", "weight_decay"):
        with pytest.raises(AttributeError, match="param_groups"):
            getattr(opt, name)
    with pytest.raises(ValueError, match="fixed at construction"):
        opt.add_param_group({"params": [nn.Parameter(torch.zeros(3))]})
    opt.zero_grad()


def test_segments_follow_the_flat_order():
    net = Net()
    opt = FlatAdam(FlatGradBucket(net.parameters()), groups=_recipe(net))
    sizes = [p.numel() for p in net.parameters()]                # emb, path, lin.weight, lin.bias, norm.weight, norm.bias
    assert opt._segments == [(0, 0), (sum(sizes[:3]), 1)]
    opt = ShardedFlatAdam([{"params": [net.emb.weight, net.lin.bias]}, {"params": [net.path.weight, net.lin.weight]},
                           {"params": [net.norm.weight, net.norm.bias], "weight_decay": 0.1}], early=[net.path.weight])
    # flat order: path (the early region, padded to 36), then emb, lin.bias, lin.weight, norm.weight, norm.bias, each
    # at a multiple of 4 elements
    assert opt.regions[1][0] == 36
    assert opt._segments == [(0, 1), (36, 0), (36 + 68 + 4, 1), (36 + 68 + 4 + 20, 2)]
    assert all(o % 4 == 0 for o in opt._flat_offsets)


@pytest.mark.parametrize("kind", KINDS)
def test_group_validation(kind):
    net = Net()
    ps = list(net.parameters())
    if kind == "flat":
        with pytest.raises(ValueError, match="exactly the bucket"):                     # a parameter missing
            _make(kind, net, [{"params": ps[:-1]}])
        with pytest.raises(ValueError, match="more than once|more than one"):          # a parameter twice
            _make(kind, net, [{"params": ps}, {"params": ps[:1]}])
    with pytest.warns(UserWarning), pytest.raises(ValueError, match="more than once"):
        _make(kind, net, [{"params": ps + ps[:1]}])
    bad = [({"max_grad_norm": 2.0}, "whole optimizer"), ({"capturable": True}, "whole optimizer"),
           ({"amsgrad": True}, "amsgrad"), ({"maximize": True}, "maximize"), ({"foreach": True}, "unknown"),
           ({"momentum": 0.9}, "unknown"), ({"lr": torch.tensor(0.01)}, "capturable=True"),
           ({"max_grad_norm": -1.0}, "max_grad_norm")]
    for extra, match in bad:
        groups = _recipe(net)
        groups[1].update(extra)
        with pytest.raises(ValueError, match=match):
            _make(kind, net, groups, max_grad_norm=1.0)
    groups = _recipe(net)
    groups[1].update(amsgrad=False, maximize=False)                  # torch's defaults are accepted
    _make(kind, net, groups)


def test_group_and_segment_limits():
    ps = [nn.Parameter(torch.zeros(3)) for _ in range(64)]
    FlatAdam(FlatGradBucket(ps), groups=[{"params": ps[k::16]} for k in range(16)])    # 16 groups, 64 runs
    with pytest.raises(ValueError, match="up to 16 groups"):
        FlatAdam(FlatGradBucket(ps), groups=[{"params": ps[k::17]} for k in range(17)])
    ps = [nn.Parameter(torch.zeros(3)) for _ in range(65)]
    with pytest.raises(ValueError, match="64 runs"):
        FlatAdam(FlatGradBucket(ps), groups=[{"params": ps[k::2]} for k in range(2)])    # 65 runs


@pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step")
@pytest.mark.parametrize("kind", KINDS)
def test_schedulers_drive_every_group(kind):
    net = Net()
    opt = _make(kind, net, _recipe(net), lr=0.1)
    sch = LS.LambdaLR(opt, [lambda e: 1.0 / (1 + e), lambda e: 0.5 ** e])
    sch.step()
    assert [g["lr"] for g in opt.param_groups] == [pytest.approx(0.05), pytest.approx(2.5e-4)]
    net = Net()
    opt = _make(kind, net, _recipe(net), lr=0.1)
    sch = LS.OneCycleLR(opt, max_lr=[1.0, 0.1], total_steps=10)
    for _ in range(2):
        sch.step()
    assert [g["lr"] for g in opt.param_groups] == [pytest.approx(1.0), pytest.approx(0.1)]
    assert all(g["betas"][0] == pytest.approx(0.85) for g in opt.param_groups)


def _torch_after(cls, net, steps, groups, **kw):
    opt = cls(groups, **kw)
    gen = torch.Generator().manual_seed(3)
    for _ in range(steps):
        for p in net.parameters():
            p.grad = torch.randn(p.shape, generator=gen)
        opt.step()
    return opt


@pytest.mark.parametrize("cls", [torch.optim.Adam, torch.optim.AdamW])
@pytest.mark.parametrize("kind", KINDS)
def test_state_dict_interchanges_with_torch(kind, cls):
    torch.manual_seed(0)
    ref_net = Net()
    ref = _torch_after(cls, ref_net, 3, _recipe(ref_net), lr=0.02)
    ref_sd = ref.state_dict()
    decoupled = cls is torch.optim.AdamW
    net = Net()
    opt = _make(kind, net, _recipe(net, wd=0.3), max_grad_norm=0.5)
    opt.load_state_dict(ref_sd)
    assert opt.t == 3 and opt.max_grad_norm is None
    assert [g["decoupled_weight_decay"] for g in opt.param_groups] == [decoupled] * 2
    assert [g["lr"] for g in opt.param_groups] == [0.02, 5e-4] and opt.param_groups[0]["weight_decay"] == 0.01
    sd = opt.state_dict()
    assert sorted(sd["state"]) == sorted(ref_sd["state"]) == list(range(6))
    assert [g["params"] for g in sd["param_groups"]] == [g["params"] for g in ref_sd["param_groups"]] == [[0, 1, 2],
                                                                                                          [3, 4, 5]]
    for a, b in zip(sd["param_groups"], ref_sd["param_groups"]):
        assert set(b) - {"foreach", "fused", "differentiable", "amsgrad", "maximize"} <= set(a)
        for k in ("lr", "betas", "eps", "weight_decay", "decoupled_weight_decay"):
            assert a[k] == b[k], k
    for i in sd["state"]:
        for k in ("step", "exp_avg", "exp_avg_sq"):
            x, y = sd["state"][i][k], ref_sd["state"][i][k]
            assert x.shape == y.shape and x.dtype == y.dtype and torch.equal(x, y), (i, k)
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    back_net = Net()
    back = cls(_recipe(back_net), lr=0.5)
    back.load_state_dict(torch.load(buf))
    assert [g["lr"] for g in back.param_groups] == [0.02, 5e-4]
    for p in back_net.parameters():
        p.grad = torch.ones_like(p)
    back.step()


@pytest.mark.parametrize("kind", KINDS)
def test_load_state_dict_errors(kind):
    net = Net()
    opt = _make(kind, net, _recipe(net))
    one = torch.optim.Adam(Net().parameters()).state_dict()
    with pytest.raises(ValueError, match=r"2 parameter groups of \[3, 3\]"):
        opt.load_state_dict(one)
    sd = _torch_after(torch.optim.Adam, n := Net(), 2, _recipe(n)).state_dict()
    sd["state"][4]["step"] = torch.tensor(1.0)
    with pytest.raises(ValueError, match="different step counts"):
        opt.load_state_dict(sd)
    sd = _torch_after(torch.optim.Adam, n := Net(), 1, _recipe(n), amsgrad=True).state_dict()
    with pytest.raises(ValueError, match="amsgrad"):
        opt.load_state_dict(sd)


# ---- the grouped entry points: C2V_EINVAL before any CUDA call ----------------------------------------------------------
def _expect_einval(rc, name):
    assert rc == _lib.C2V_EINVAL
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


def _table(n_groups=2, seg_begin=(0, 5), seg_group=(0, 1), n_segments=None, lr_dev=None):
    groups = (_lib.AdamGroup * max(n_groups, 1))()
    for g in groups:
        g.lr, g.beta1, g.beta2, g.eps, g.weight_decay, g.decoupled, g.lr_dev = 1e-3, 0.9, 0.999, 1e-8, 0.0, 0, lr_dev
    n_segments = len(seg_begin) if n_segments is None else n_segments
    return (groups, n_groups, (ctypes.c_int64 * max(len(seg_begin), 1))(*seg_begin),
            (ctypes.c_int32 * max(len(seg_group), 1))(*seg_group), n_segments)


TABLE_BAD = {"zero groups": dict(n_groups=0), "17 groups": dict(n_groups=17), "zero segments": dict(n_segments=0),
             "65 segments": dict(seg_begin=range(65), seg_group=[0] * 65),
             "first segment not at 0": dict(seg_begin=(4, 8)), "unsorted": dict(seg_begin=(0, 9, 5), seg_group=(0, 1, 0)),
             "overlapping": dict(seg_begin=(0, 5, 5), seg_group=(0, 1, 0)),
             "group out of range": dict(seg_group=(0, 2)), "negative group": dict(seg_group=(-1, 0))}


def _flat(table, state=None, step=1):
    return _lib.load().c2v_adam_step_groups(FAKE, FAKE, FAKE, FAKE, 100, *table, step, state, 1.0, 1, None, None)


@pytest.mark.parametrize("case", list(TABLE_BAD))
def test_grouped_entry_points_reject_bad_tables(case):
    t = _table(**TABLE_BAD[case])
    _expect_einval(_flat(t), "c2v_adam_step_groups")
    pt = (V * 2)(FAKE, FAKE)
    rc = _lib.load().c2v_adam_step_sharded_groups(FAKE, None, None, pt, pt, 2, FAKE, FAKE, 0, 64, None, 0, *t, 1, 0.5,
                                                   None)
    _expect_einval(rc, "c2v_adam_step_sharded_groups")
    rc = _lib.load().c2v_adam_step_sharded_bulk_groups(FAKE, pt, pt, 2, FAKE, FAKE, 0, 64, *t, 1, 0.5, 0, None)
    _expect_einval(rc, "c2v_adam_step_sharded_bulk_groups")


def test_grouped_flat_step_rejects_bad_arguments():
    _expect_einval(_flat(_table(), step=0), "c2v_adam_step_groups")                 # host step < 1
    _expect_einval(_flat(_table(lr_dev=FAKE)), "c2v_adam_step_groups")              # lr_dev without step_state
    _expect_einval(_flat(_table(lr_dev=V(0x1001)), state=FAKE), "c2v_adam_step_groups")
    _expect_einval(_flat(_table(), state=V(0x1004)), "c2v_adam_step_groups")        # misaligned step_state
    rc = _lib.load().c2v_adam_step_groups(FAKE, FAKE, ODD, FAKE, 100, *_table(), 1, None, 1.0, 1, None, None)
    _expect_einval(rc, "c2v_adam_step_groups")
    pt = (V * 2)(FAKE, FAKE)
    rc = _lib.load().c2v_adam_step_sharded_groups(FAKE, None, None, pt, pt, 2, FAKE, FAKE, 2, 64, None, 0, *_table(), 1,
                                                   0.5, None)
    _expect_einval(rc, "c2v_adam_step_sharded_groups")                             # slice_begin % 4
