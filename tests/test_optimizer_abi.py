"""CPU-side checks of FlatAdam / ShardedFlatAdam as torch optimizers: the argument errors of c2v_grad_clip_coef and
c2v_adam_step_ex return C2V_EINVAL before any CUDA call (without a GPU a CUDA call would return C2V_ECUDA), the
lr_scheduler classes drive the one parameter group, and state_dict() / load_state_dict() interchange with
torch.optim.Adam's.  Nothing here launches a kernel: the optimizers are built over CPU parameters and never stepped."""
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
ODD = V(0x1004)           # 4-byte aligned, not 16-byte aligned
BYTE = V(0x1001)


def _expect_einval(rc, name):
    assert rc == _lib.C2V_EINVAL
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


def _clip(g=FAKE, n=100, max_norm=1.0, out=FAKE, ws=FAKE, ws_bytes=1 << 20):
    return _lib.load().c2v_grad_clip_coef(g, n, 1.0, max_norm, out, ws, ws_bytes, None)


CLIP_BAD = {"grad": dict(g=None), "out": dict(out=None), "workspace": dict(ws=None), "n<1": dict(n=0), "n<0": dict(n=-8),
            "max_norm 0": dict(max_norm=0.0), "max_norm<0": dict(max_norm=-1.0), "max_norm NaN": dict(max_norm=float("nan")),
            "misaligned grad": dict(g=ODD), "misaligned out": dict(out=BYTE), "misaligned workspace": dict(ws=BYTE),
            "small workspace": dict(n=10 ** 6, ws_bytes=64), "no workspace bytes": dict(ws_bytes=0)}


@pytest.mark.parametrize("case", list(CLIP_BAD))
def test_grad_clip_coef_rejects_bad_arguments(case):
    _expect_einval(_clip(**CLIP_BAD[case]), "c2v_grad_clip_coef")


def test_grad_norm_workspace_bytes_positive_and_monotone():
    f = _lib.load().c2v_grad_norm_workspace_bytes
    assert f(0) == 0 and f(-5) == 0
    sizes = [1, 3, 4, 1023, 1024, 1025, 10 ** 5, 10 ** 6, 2 * 10 ** 6, 9 * 10 ** 7, 10 ** 10]
    got = [f(n) for n in sizes]
    assert all(b > 0 and b % 4 == 0 for b in got) and got == sorted(got)
    assert got[-1] == got[-2] == 4096                       # the grid, and with it the workspace, is capped
    assert _clip(n=10 ** 6, ws_bytes=f(10 ** 6) - 4) == _lib.C2V_EINVAL


def _ex(p=FAKE, g=FAKE, m=FAKE, v=FAKE, n=100, step=1, state=None, lr_dev=None, coef_dev=None):
    return _lib.load().c2v_adam_step_ex(p, g, m, v, n, 1e-3, 0.9, 0.999, 1e-8, 0.0, step, state, 1.0, 1, lr_dev, coef_dev,
                                        None)


EX_BAD = {"param": dict(p=None), "grad": dict(g=None), "exp_avg": dict(m=None), "exp_avg_sq": dict(v=None),
          "n<1": dict(n=0), "misaligned param": dict(p=ODD), "misaligned exp_avg_sq": dict(v=ODD),
          "host step<1": dict(step=0), "host step<1 with coef": dict(step=0, coef_dev=FAKE),
          "misaligned step_state": dict(state=ODD), "lr_dev without step_state": dict(lr_dev=FAKE),
          "misaligned lr_dev": dict(state=FAKE, lr_dev=BYTE), "misaligned coef_dev": dict(coef_dev=BYTE),
          "misaligned coef_dev, device step": dict(state=FAKE, coef_dev=V(0x1002))}


@pytest.mark.parametrize("case", list(EX_BAD))
def test_adam_step_ex_rejects_bad_arguments(case):
    _expect_einval(_ex(**EX_BAD[case]), "c2v_adam_step_ex")


# ---- the optimizers as torch.optim.Optimizers ------------------------------------------------------------------------
class Net(nn.Module):
    """four parameters of different shapes; `path` stands for the table ShardedFlatAdam(early=...) moves to the front"""

    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(11, 6)
        self.path = nn.Embedding(7, 5)
        self.lin = nn.Linear(6, 3)


def _make(kind, net, **kw):
    if kind == "flat":
        return FlatAdam(FlatGradBucket(net.parameters()), **kw)
    if kind == "sharded":
        return ShardedFlatAdam(net.parameters(), **kw)
    return ShardedFlatAdam(net.parameters(), early=[net.path.weight], **kw)


KINDS = ["flat", "sharded", "sharded-early"]


@pytest.mark.parametrize("kind", KINDS)
def test_is_a_torch_optimizer_with_one_group(kind):
    net = Net()
    opt = _make(kind, net, lr=0.02, betas=(0.8, 0.99), eps=1e-7, weight_decay=0.1, max_grad_norm=2.0)
    assert isinstance(opt, torch.optim.Optimizer) and len(opt.param_groups) == 1
    g = opt.param_groups[0]
    assert [id(p) for p in g["params"]] == [id(p) for p in net.parameters()]          # the caller's order
    assert (g["lr"], g["betas"], g["eps"], g["weight_decay"], g["max_grad_norm"], g["capturable"]) == \
        (0.02, (0.8, 0.99), 1e-7, 0.1, 2.0, False)
    assert (opt.lr, opt.betas, opt.eps, opt.weight_decay, opt.max_grad_norm, opt.capturable) == \
        (0.02, (0.8, 0.99), 1e-7, 0.1, 2.0, False)
    g["lr"] = 0.5                                            # the group is the source of truth ...
    assert opt.lr == 0.5
    opt.weight_decay = 0.0                                   # ... and the attributes write it
    assert g["weight_decay"] == 0.0
    assert opt.grad_norm.shape == (1,) and opt.grad_norm.dtype == torch.float32
    with pytest.raises(ValueError, match="one parameter group"):
        opt.add_param_group({"params": [nn.Parameter(torch.zeros(3))]})
    opt.zero_grad()
    assert all(p.grad is not None for p in net.parameters())


@pytest.mark.filterwarnings("ignore:Detected call of `lr_scheduler.step")
@pytest.mark.parametrize("kind", KINDS)
def test_lr_schedulers_drive_the_group(kind):
    opt = _make(kind, Net(), lr=0.1)
    sch = LS.LambdaLR(opt, lambda e: 1.0 / (1 + e))
    sch.step()
    assert opt.lr == opt.param_groups[0]["lr"] == pytest.approx(0.05)
    opt = _make(kind, Net(), lr=0.1)
    sch = LS.StepLR(opt, step_size=2, gamma=0.1)
    for _ in range(2):
        sch.step()
    assert opt.lr == pytest.approx(0.01)
    opt = _make(kind, Net(), lr=0.1)
    sch = LS.CosineAnnealingLR(opt, T_max=4)
    for _ in range(4):
        sch.step()
    assert opt.lr == pytest.approx(0.0, abs=1e-9)
    opt = _make(kind, Net(), lr=0.1)
    sch = LS.ReduceLROnPlateau(opt, factor=0.5, patience=0)
    sch.step(1.0)
    sch.step(2.0)
    assert opt.lr == pytest.approx(0.05)
    opt = _make(kind, Net(), lr=0.1)
    sch = LS.OneCycleLR(opt, max_lr=1.0, total_steps=10)      # cycles betas[0] as well
    assert opt.lr == pytest.approx(0.04) and opt.betas == (0.95, 0.999)
    for _ in range(2):
        sch.step()
    assert opt.lr == pytest.approx(1.0) and opt.betas[0] == pytest.approx(0.85) and opt.betas[1] == 0.999


@pytest.mark.parametrize("kind", KINDS)
def test_constructor_errors(kind):
    with pytest.raises(ValueError, match="capturable=True"):
        _make(kind, Net(), lr=torch.tensor(0.01))
    for bad in (0.0, -1.0, float("nan")):
        with pytest.raises(ValueError, match="max_grad_norm"):
            _make(kind, Net(), max_grad_norm=bad)


def test_tensor_lr_must_be_one_fp32_element_on_the_parameters_device():
    net = Net()
    for lr in (torch.tensor(0.01, dtype=torch.float64), torch.tensor([0.01, 0.02]), torch.tensor(0.01, device="meta")):
        with pytest.raises(ValueError, match="one-element fp32"):
            FlatAdam(FlatGradBucket(net.parameters()), lr=lr, capturable=True)


def test_sharded_max_grad_norm_needs_world_one(monkeypatch):
    import torch.distributed as dist
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    with pytest.raises(NotImplementedError, match="one process"):
        ShardedFlatAdam(Net().parameters(), max_grad_norm=1.0)


# ---- state_dict ------------------------------------------------------------------------------------------------------
def _torch_adam_after(net, steps, **kw):
    opt = torch.optim.Adam(net.parameters(), **kw)
    g = torch.Generator().manual_seed(3)
    for _ in range(steps):
        for p in net.parameters():
            p.grad = torch.randn(p.shape, generator=g)
        opt.step()
    return opt


@pytest.mark.parametrize("kind", KINDS)
def test_state_dict_has_torch_adams_layout_and_round_trips(kind):
    torch.manual_seed(0)
    ref_net = Net()
    ref = _torch_adam_after(ref_net, 3, lr=0.02, weight_decay=0.01)
    ref_sd = ref.state_dict()
    net = Net()
    opt = _make(kind, net, max_grad_norm=0.5)
    opt.load_state_dict(ref_sd)                              # torch's dict loads ...
    assert opt.t == opt.step_count() == 3 and opt.lr == 0.02 and opt.weight_decay == 0.01 and opt.max_grad_norm is None
    sd = opt.state_dict()
    assert sorted(sd) == sorted(ref_sd) and sorted(sd["state"]) == sorted(ref_sd["state"]) == [0, 1, 2, 3]
    assert sd["param_groups"][0]["params"] == ref_sd["param_groups"][0]["params"] == [0, 1, 2, 3]
    for i, p in enumerate(net.parameters()):
        a, b = sd["state"][i], ref_sd["state"][i]
        assert sorted(a) == sorted(b) == ["exp_avg", "exp_avg_sq", "step"]
        for k in a:                                          # ... and comes back with the same keys, shapes, dtypes, values
            assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype and a[k].device == b[k].device, (i, k)
            assert torch.equal(a[k], b[k]), (i, k)
        assert a["exp_avg"].shape == p.shape
    flat = opt.exp_avg
    sd["state"][0]["exp_avg"].add_(1.0)                      # copies, not views of the flat buffers
    assert torch.equal(flat, opt.exp_avg.clone()) and not torch.equal(opt.state_dict()["state"][0]["exp_avg"],
                                                                      sd["state"][0]["exp_avg"])
    sd = opt.state_dict()
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    again = _make(kind, Net(), lr=0.5, max_grad_norm=3.0)
    again.load_state_dict(torch.load(buf))
    assert torch.equal(again.exp_avg, opt.exp_avg) and torch.equal(again.exp_avg_sq, opt.exp_avg_sq)
    assert again.t == 3 and again.lr == 0.02 and again.max_grad_norm is None
    # torch's Adam loads ours and continues
    back = torch.optim.Adam(Net().parameters())
    back.load_state_dict(sd)
    assert back.param_groups[0]["lr"] == 0.02 and float(back.state[back.param_groups[0]["params"][2]]["step"]) == 3.0
    for p in back.param_groups[0]["params"]:
        p.grad = torch.ones_like(p)
    back.step()


def test_early_parameters_keep_the_callers_order_in_the_state_dict():
    net = Net()
    opt = ShardedFlatAdam(net.parameters(), early=[net.path.weight])
    assert opt.params[0] is net.path.weight and opt._flat_offsets[1] == 0        # flat order: the early table first
    n = net.path.weight.numel()
    opt.exp_avg[:n] = 7.0
    sd = opt.state_dict()
    assert float(sd["state"][1]["exp_avg"].min()) == 7.0 and sd["state"][1]["exp_avg"].shape == net.path.weight.shape
    assert all(float(sd["state"][i]["exp_avg"].abs().max()) == 0.0 for i in (0, 2, 3))


@pytest.mark.parametrize("kind", KINDS)
def test_fresh_and_frozen_states(kind):
    opt = _make(kind, Net())
    opt.exp_avg.fill_(1.0)
    opt.t = 5
    opt.load_state_dict(torch.optim.Adam(Net().parameters(), lr=0.3).state_dict())     # no state yet: zeros, step 0
    assert opt.t == 0 and float(opt.exp_avg.abs().max()) == 0.0 and opt.lr == 0.3
    net = Net()
    sd = _torch_adam_after(net, 2).state_dict()
    sd["state"][1]["step"] = torch.tensor(1.0)               # a parameter that sat out a step
    with pytest.raises(ValueError, match="different step counts"):
        opt.load_state_dict(sd)
    sd = _torch_adam_after(Net(), 2, amsgrad=True).state_dict()
    with pytest.raises(ValueError, match="amsgrad"):
        opt.load_state_dict(sd)
    sd = _torch_adam_after(Net(), 1).state_dict()
    sd["param_groups"][0]["params"] = [0, 1, 2]
    with pytest.raises(ValueError, match="one parameter group of 4"):
        opt.load_state_dict(sd)
